// vision_kernels.cuh — sm_90a kernels of the vision graph (EVA ViT-g/14 + Q-Former + llama_proj), the path
// behind minigpt4_encode_image (reference minigpt4.cpp:2094-2363).
//
// Dense contractions run on the Hopper tensor cores: a producer warp stages F16 operand tiles in shared memory with TMA
// (cp.async.bulk.tensor, 128B swizzle), two consumer warpgroups issue wgmma.mma_async m64nNk16 (both operands read from
// shared memory, F32 accumulator in registers) and then fuse bias / GELU / residual / positional-embedding work on it.
// ggml numerics (SURVEY §A.3): F16 weights x activations rounded to F16, F32 accumulation — exactly f32.f16.f16.
//
// "Swap-AB" tiling: wgmma M (2 x 64) runs over OUTPUT FEATURES (always a multiple of 128 here), wgmma N over TOKENS
// (one instruction shape per token tile: 32, 80, 144 or 256), so each CTA streams its weight slab exactly once.
#pragma once
#include "common.h"
#include <cuda.h>

namespace mg4 {
namespace vk {

enum GemmEpi : int { GE_BIAS = 0, GE_QSCALE = 1, GE_GELU_F16 = 2, GE_RESID = 3, GE_PATCH = 4, GE_PARTIAL = 5 /* split-K kernel only */ };

struct GemmArgs {
    int M_out, T, K;          // output features (multiple of 128), valid tokens, contraction (multiple of 64)
    int nt;                   // tokens per CTA = wgmma N (32, 80, 144 or 256); grid.y = ceil(T / nt)
    int stages, stage_bytes;
    int epi;
    const float *bias;        // [M_out] or null
    float qscale; int qscale_rows;  // GE_QSCALE: rows < qscale_rows are multiplied by qscale after the bias
    float *out_f32; __half *out_f16; int ld_out;
    const float *resid;       // GE_RESID: out = resid + (acc + bias)   (may alias out_f32)
    const float *pos;         // GE_PATCH: out[t+1] = acc + bias + pos[t+1]
    const __half *tab_gelu;
    int k_split_blocks;       // split-K: 64-wide k-blocks per grid.z slice (0: no split)
    float *partial; long long partial_stride;  // GE_PARTIAL: slice z writes acc (+ bias if z == 0) to partial[z * partial_stride + t * ld_out + m]
};

constexpr int kGemmThreads = 288;   // warps 0-7 = two consumer warpgroups (64 features each), warp 8 = TMA producer

// ---- raw PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 format: layout type 1 in bits 62-63, SBO = 8 rows * 128 B; LBO unused)
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, F16 operands from shared memory, F32 accumulator: thread (warp w, lane) of the warpgroup holds
// d[4 j + 2 h + e] = D[16 w + lane / 4 + 8 h][8 j + 2 (lane % 4) + e]
__device__ __forceinline__ void wgmma_f16(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16(float (&d)[40], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16(float (&d)[72], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %74, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n144k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71}, %72, %73, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_f16(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
                 : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
// ---------------------------------------------------------------------------------------------
// out[t][m] = epi( sum_k W[m][k] * X[t][k] )      W: F16 [M_out][K] (TMA map tmW), X: F16 [T][K] (TMA map tmX)
// grid.x = M_out/128 CTAs of 288 threads: warps 0-7 = two consumer warpgroups (wgmma + epilogue, 64 features each), warp 8 = TMA producer
// ---------------------------------------------------------------------------------------------
// TOKEN SPLIT (grid.y): the CTAs of one 128-feature weight slab take NT tokens each, so the T = 257 GEMMs spread over most of the SMs instead
// of 11-48 of them; rows past T come back from TMA as zeros and are masked in the epilogue.
// SPLIT-K (grid.z, the two residual GEMMs proj / fc2 whose M is only 1408): a CTA covers the k-blocks [z * k_split_blocks, ...) of its tile and
// writes raw partial sums (GE_PARTIAL, bias on slice 0); layernorm_fold_kernel folds the slices into the residual stream in slice order
// (deterministic).
template <int NT>
__global__ void __launch_bounds__(kGemmThreads, 1) gemm_f16_wgmma(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const GemmArgs g) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *full = (uint64_t *)(smem + (size_t)g.stages * g.stage_bytes);
    uint64_t *empty = full + 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_tile = blockIdx.x;
    const int t0 = (int)blockIdx.y * NT;  // first token of this CTA
    const int num_k_all = g.K / 64;
    const int kb0 = (g.k_split_blocks != 0) ? (int)blockIdx.z * g.k_split_blocks : 0;          // first k-block of this CTA (split-K)
    const int num_k = (g.k_split_blocks != 0) ? min(g.k_split_blocks, num_k_all - kb0) : num_k_all;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmX) : "memory");
        for (int i = 0; i < g.stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }   // a stage is free when the 8 consumer warps have released it
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            const uint32_t tx = 16384u + (uint32_t)NT * 128u;
            for (int kb = 0; kb < num_k; ++kb) {
                const int s = kb % g.stages; const uint32_t ph = (uint32_t)(kb / g.stages) & 1u;
                mbar_wait(&empty[s], ph ^ 1u);
                unsigned char *sa = smem + (size_t)s * g.stage_bytes, *sb = sa + 16384;
                mbar_expect_tx(&full[s], tx);
                tma_load_2d(sa, &tmW, (kb0 + kb) * 64, m_tile * 128, &full[s]);
                tma_load_2d(sb, &tmX, (kb0 + kb) * 64, t0, &full[s]);
            }
        }
        return;
    }
    const int wg = warp >> 2;
    float acc[NT / 2];
    for (int kb = 0; kb < num_k; ++kb) {
        const int s = kb % g.stages; const uint32_t ph = (uint32_t)(kb / g.stages) & 1u;
        mbar_wait(&full[s], ph);
        const uint32_t sa = smem_u32(smem + (size_t)s * g.stage_bytes) + (uint32_t)wg * 8192u, sb = sa - (uint32_t)wg * 8192u + 16384u;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_f16(acc, wgmma_desc_sw128(sa + k * 32), wgmma_desc_sw128(sb + k * 32), (uint32_t)((kb | k) != 0));
        wgmma_commit();
        if (kb > 0) {   // one k-block stays in flight: the tensor core has finished reading the previous stage
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(&empty[(kb - 1) % g.stages]);
        }
    }
    wgmma_wait<0>();

    const int m0 = m_tile * 128 + wg * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's features: m0 and m0 + 8
    const int tl = t0 + 2 * (lane & 3);                                      // ... and tokens: tl + 8 j + {0, 1}
    float bias[2], qs[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        bias[h] = g.bias ? g.bias[m0 + 8 * h] : 0.f;
        qs[h] = (g.epi == GE_QSCALE && m0 + 8 * h < g.qscale_rows) ? g.qscale : 1.0f;
    }
    // batches of 16 accumulators (four 8-token chunks): value q of a batch is chunk q / 4, feature half (q / 2) % 2, token q % 2
#pragma unroll
    for (int jb = 0; jb < NT / 8; jb += 4) {
        if (g.epi == GE_PARTIAL) {  // split-K slice: raw partial sums (bias rides on slice 0); the following LayerNorm folds the slices into x
            float *dst = g.partial + (size_t)blockIdx.z * (size_t)g.partial_stride;
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int j = jb + (q >> 2), h = (q >> 1) & 1, t = tl + 8 * j + (q & 1);
                if (j < NT / 8 && t < g.T) dst[(size_t)t * g.ld_out + m0 + 8 * h] = (blockIdx.z == 0 ? bias[h] : 0.f) + acc[(j < NT / 8 ? j : 0) * 4 + (q & 3)];
            }
            continue;
        }
        // No early exit inside the batch: every load of the batch (residual / positional embedding) is issued
        // before its first use, so the epilogue pays one L2 round trip per batch instead of one per token.
        float aux[16];
        if (g.epi == GE_RESID || g.epi == GE_PATCH) {
            const float *src = g.epi == GE_RESID ? g.resid : g.pos;
            const int off = g.epi == GE_PATCH ? 1 : 0;
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int j = jb + (q >> 2), h = (q >> 1) & 1, t = tl + 8 * j + (q & 1);
                aux[q] = (j < NT / 8 && t < g.T) ? src[(size_t)(t + off) * g.ld_out + m0 + 8 * h] : 0.f;
            }
        }
        if (g.epi == GE_GELU_F16) {
            __half hv[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int j = jb + (q >> 2), h = (q >> 1) & 1;
                hv[q] = g.tab_gelu[__half_as_ushort(__float2half_rn(bias[h] + acc[(j < NT / 8 ? j : 0) * 4 + (q & 3)]))];
            }
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int j = jb + (q >> 2), h = (q >> 1) & 1, t = tl + 8 * j + (q & 1);
                if (j < NT / 8 && t < g.T) g.out_f16[(size_t)t * g.ld_out + m0 + 8 * h] = hv[q];
            }
            continue;
        }
#pragma unroll
        for (int q = 0; q < 16; ++q) {
            const int j = jb + (q >> 2), h = (q >> 1) & 1, t = tl + 8 * j + (q & 1), m = m0 + 8 * h;
            if (j < NT / 8 && t < g.T) {
                float r = bias[h] + acc[(j < NT / 8 ? j : 0) * 4 + (q & 3)];
                switch (g.epi) {
                    case GE_QSCALE: r *= qs[h]; g.out_f32[(size_t)t * g.ld_out + m] = r; break;
                    case GE_RESID: g.out_f32[(size_t)t * g.ld_out + m] = aux[q] + r; break;
                    case GE_PATCH: g.out_f32[(size_t)(t + 1) * g.ld_out + m] = (0.0f + r) + aux[q]; break;
                    default: g.out_f32[(size_t)t * g.ld_out + m] = r; if (g.out_f16) g.out_f16[(size_t)t * g.ld_out + m] = __float2half_rn(r); break;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (ggml_norm eps 1e-5 with double accumulation, then w*x+b): F32 rows -> F16 (GEMM operand) and/or F32
// one warp per row
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
// one CTA of 128 threads per row (n <= 1536: 12 values per thread, in registers, one global pass).  A single warp per row made the
// kernel a ~1900-instruction dependent chain with one warp per scheduler; four warps per row
// cut the chain by 4 and give every scheduler of every SM something to overlap.
__global__ void __launch_bounds__(128) layernorm_kernel(const float *__restrict__ x, int rows, int n, const float *__restrict__ w, const float *__restrict__ b,
                                                        __half *__restrict__ out16, float *__restrict__ out32, const float *__restrict__ add_in /* optional: x + add_in before the norm */) {
    __shared__ double red[8];
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (row >= rows) return;
    const float *xr = x + (size_t)row * n;
    const float *ar = add_in ? add_in + (size_t)row * n : nullptr;
    constexpr int MAXE = 12;
    float v[MAXE];
#pragma unroll
    for (int k = 0; k < MAXE; ++k) {
        const int i = tid + 128 * k, ic = min(i, n - 1);  // clamped, unconditional loads; out-of-range slots hold 0
        const float t = ar ? xr[ic] + ar[ic] : xr[ic];
        v[k] = i < n ? t : 0.f;
    }
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < MAXE; ++k) s += (double)v[k];
    s = warp_sum_d(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    s = (red[0] + red[1]) + (red[2] + red[3]);
    const float mean = (float)(s / (double)n);
    double s2 = 0.0;
#pragma unroll
    for (int k = 0; k < MAXE; ++k) { v[k] = v[k] - mean; if (tid + 128 * k < n) s2 += (double)(v[k] * v[k]); }
    s2 = warp_sum_d(s2);
    if (lane == 0) red[4 + warp] = s2;
    __syncthreads();
    s2 = (red[4] + red[5]) + (red[6] + red[7]);
    const float variance = (float)(s2 / (double)n);
    const float scale = 1.0f / sqrtf(variance + 1e-5f);
#pragma unroll
    for (int k = 0; k < MAXE; ++k) {
        const int i = tid + 128 * k;
        if (i < n) {
            float y = w[i] * (v[k] * scale);
            if (b) y = y + b[i];
            if (out16) out16[(size_t)row * n + i] = __float2half_rn(y);
            if (out32) out32[(size_t)row * n + i] = y;
        }
    }
}

// LayerNorm that first folds split-K partial sums into the residual stream (GE_PARTIAL): t = ((x + p0) + p1) + ... in
// slice order (deterministic), written back to x, then normalised exactly like layernorm_kernel.  One CTA of 128 threads per row.
__global__ void __launch_bounds__(128) layernorm_fold_kernel(float *__restrict__ x, int rows, int n, const float *__restrict__ w, const float *__restrict__ b,
                                                             __half *__restrict__ out16, const float *__restrict__ parts, int n_parts, long long part_stride) {
    __shared__ double red[8];
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (row >= rows) return;
    float *xr = x + (size_t)row * n;
    constexpr int MAXE = 12;
    float v[MAXE];
#pragma unroll
    for (int k = 0; k < MAXE; ++k) {
        const int i = tid + 128 * k, ic = min(i, n - 1);
        float t = xr[ic];
        for (int p = 0; p < n_parts; ++p) t = t + parts[(size_t)p * (size_t)part_stride + (size_t)row * n + ic];
        if (i < n) xr[i] = t;
        v[k] = i < n ? t : 0.f;
    }
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < MAXE; ++k) s += (double)v[k];
    s = warp_sum_d(s);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    s = (red[0] + red[1]) + (red[2] + red[3]);
    const float mean = (float)(s / (double)n);
    double s2 = 0.0;
#pragma unroll
    for (int k = 0; k < MAXE; ++k) { v[k] = v[k] - mean; if (tid + 128 * k < n) s2 += (double)(v[k] * v[k]); }
    s2 = warp_sum_d(s2);
    if (lane == 0) red[4 + warp] = s2;
    __syncthreads();
    s2 = (red[4] + red[5]) + (red[6] + red[7]);
    const float variance = (float)(s2 / (double)n);
    const float scale = 1.0f / sqrtf(variance + 1e-5f);
#pragma unroll
    for (int k = 0; k < MAXE; ++k) {
        const int i = tid + 128 * k;
        if (i < n) { float y = w[i] * (v[k] * scale); if (b) y = y + b[i]; out16[(size_t)row * n + i] = __float2half_rn(y); }
    }
}

// ---------------------------------------------------------------------------------------------
// F32 multi-head attention (ViT MHSA and Q-Former self/cross attention; ggml F32xF32 mul_mat + soft_max with fp16 exp LUT)
// q: [nq][ldq] (+ head*DH), k,v: [nk][ldkv] (+ head*DH).  grid (heads, ceil(nq / q_per_cta)), block 256.
// K ([nk][DH+4], float4 rows, odd float4 pitch -> conflict-free 128-bit reads) and V ([nk][DH]) of the head live in shared
// memory.  The kernel is shared-memory-bandwidth bound, so each warp processes NQ = 4 queries at a time: every K / V value read from
// shared memory feeds 4 FMAs.  The per-warp
// scratch holds the warp's q rows while the scores are formed and is then reused for its probability rows.  Per element the
// arithmetic (FMA order over d and over keys, LUT exp, double sum) is unchanged.  out: F16 [nq][ld_out] (operand of the next GEMM).
// ---------------------------------------------------------------------------------------------
constexpr int kAttnNQ = 4;
template <int DH>
__global__ void __launch_bounds__(256) attention_f32_kernel(const float *__restrict__ q, int ldq, const float *__restrict__ k, const float *__restrict__ v, int ldkv,
                                                            int nq, int nk, float score_div, int q_per_cta, __half *__restrict__ out, int ld_out,
                                                            const __half *__restrict__ tab_exp) {
    extern __shared__ __align__(16) unsigned char smem[];
    constexpr int DH4 = DH / 4, KP = DH + 4, NKI = 9, NQ = kAttnNQ;  // nk <= 288
    const int nk_pad = (nk + 31) & ~31;
    const int wstride = NQ * (nk_pad > DH ? nk_pad : DH);
    float *Ks = (float *)smem; float *Vs = Ks + (size_t)nk * KP; float *Ws = Vs + (size_t)nk * DH;
    const int h = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int t = warp; t < nk; t += 8) {
        if (lane < DH4) {
            *(float4 *)(Ks + (size_t)t * KP + lane * 4) = *(const float4 *)(k + (size_t)t * ldkv + h * DH + lane * 4);
            *(float4 *)(Vs + (size_t)t * DH + lane * 4) = *(const float4 *)(v + (size_t)t * ldkv + h * DH + lane * 4);
        }
    }
    __syncthreads();
    const int q0 = blockIdx.y * q_per_cta, q1 = min(nq, q0 + q_per_cta);
    float *qw = Ws + (size_t)warp * wstride, *pw = qw;
    for (int tq = q0 + NQ * warp; tq < q1; tq += 8 * NQ) {
        const int nv = min(NQ, q1 - tq);  // valid queries of this pass (the others are computed on zeros and dropped)
        if (lane < DH4) {
#pragma unroll
            for (int qi = 0; qi < NQ; ++qi)
                *(float4 *)(qw + qi * DH + lane * 4) = qi < nv ? *(const float4 *)(q + (size_t)(tq + qi) * ldq + h * DH + lane * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        __syncwarp();
        float sc[NQ][NKI];
#pragma unroll
        for (int qi = 0; qi < NQ; ++qi)
#pragma unroll
            for (int i = 0; i < NKI; ++i) sc[qi][i] = 0.f;
        for (int c = 0; c < DH4; ++c) {
            float4 qv[NQ];
#pragma unroll
            for (int qi = 0; qi < NQ; ++qi) qv[qi] = *(const float4 *)(qw + qi * DH + c * 4);
#pragma unroll
            for (int i = 0; i < NKI; ++i) {
                const int j = min(lane + 32 * i, nk - 1);  // clamped: lanes past the last key compute a value that is never used
                const float4 kk = *(const float4 *)(Ks + (size_t)j * KP + c * 4);
#pragma unroll
                for (int qi = 0; qi < NQ; ++qi) {
                    sc[qi][i] = fmaf(kk.x, qv[qi].x, sc[qi][i]); sc[qi][i] = fmaf(kk.y, qv[qi].y, sc[qi][i]);
                    sc[qi][i] = fmaf(kk.z, qv[qi].z, sc[qi][i]); sc[qi][i] = fmaf(kk.w, qv[qi].w, sc[qi][i]);
                }
            }
        }
        __syncwarp();  // every lane has finished reading the q rows: the scratch becomes the probability rows
#pragma unroll
        for (int qi = 0; qi < NQ; ++qi) {
            float mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < NKI; ++i) if (lane + 32 * i < nk) { sc[qi][i] = sc[qi][i] / score_div; mx = fmaxf(mx, sc[qi][i]); }
            mx = warp_max_f(mx);
            double sum = 0.0;
#pragma unroll
            for (int i = 0; i < NKI; ++i) if (lane + 32 * i < nk) {
                sc[qi][i] = __half2float(tab_exp[__half_as_ushort(__float2half_rn(sc[qi][i] - mx))]); sum += (double)sc[qi][i];
            }
            sum = warp_sum_d(sum);
            const float inv = (float)(1.0 / sum);
#pragma unroll
            for (int i = 0; i < NKI; ++i) { const int j = lane + 32 * i; if (j < nk_pad) pw[qi * nk_pad + j] = j < nk ? sc[qi][i] * inv : 0.f; }
        }
        __syncwarp();
        float o[NQ][3];
#pragma unroll
        for (int qi = 0; qi < NQ; ++qi) { o[qi][0] = 0.f; o[qi][1] = 0.f; o[qi][2] = 0.f; }
        for (int j4 = 0; j4 < nk_pad; j4 += 4) {
            float pv[NQ][4];
#pragma unroll
            for (int qi = 0; qi < NQ; ++qi) { const float4 p4 = *(const float4 *)(pw + qi * nk_pad + j4); pv[qi][0] = p4.x; pv[qi][1] = p4.y; pv[qi][2] = p4.z; pv[qi][3] = p4.w; }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int j = j4 + u;
                if (j < nk) {
#pragma unroll
                    for (int e = 0; e < 3; ++e) {
                        const int d = lane + 32 * e;
                        if (d < DH) {
                            const float vv = Vs[(size_t)j * DH + d];
#pragma unroll
                            for (int qi = 0; qi < NQ; ++qi) o[qi][e] = fmaf(vv, pv[qi][u], o[qi][e]);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int qi = 0; qi < NQ; ++qi) {
            if (qi < nv) {
#pragma unroll
                for (int e = 0; e < 3; ++e) { const int d = lane + 32 * e; if (d < DH) out[(size_t)(tq + qi) * ld_out + h * DH + d] = __float2half_rn(o[qi][e]); }
            }
        }
        __syncwarp();
    }
}

// im2col for the 14x14/stride-14 patch embedding: image F32 CHW [3][224][224] -> F16 [256][kpad] with
// column = ic*196 + ky*14 + kx (ggml_conv_2d_sk_p0 order), zero padded to kpad
__global__ void im2col_patch_kernel(const float *__restrict__ img, __half *__restrict__ out, int kpad) {
    const int p = blockIdx.x, oy = p / 16, ox = p % 16;
    for (int c = threadIdx.x; c < kpad; c += blockDim.x) {
        float v = 0.f;
        if (c < 588) { const int ic = c / 196, ky = (c % 196) / 14, kx = c % 14; v = img[(size_t)ic * 224 * 224 + (size_t)(oy * 14 + ky) * 224 + ox * 14 + kx]; }
        out[(size_t)p * kpad + c] = __float2half_rn(v);
    }
}
__global__ void cls_row_kernel(const float *__restrict__ cls, const float *__restrict__ pos, float *__restrict__ x, int D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < D) x[i] = (0.0f + cls[i]) + pos[i];
}
__global__ void f32_to_f16_kernel(const float *__restrict__ in, __half *__restrict__ out, size_t n) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = __float2half_rn(in[i]);
}
__global__ void pad_rows_f16_kernel(const __half *__restrict__ src, int rows, int cols, __half *__restrict__ dst, int dst_cols) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)rows * dst_cols) return;
    const int r = (int)(i / dst_cols), c = (int)(i % dst_cols);
    dst[i] = c < cols ? src[(size_t)r * cols + c] : __float2half_rn(0.f);
}

// Load-time conversion of a non-F16 matrix to the F16 operand layout of the tensor-core path: F32, or ggml's 32-element block
// types (what minigpt4_quantize_model can produce for a ViT-g / Q-Former matrix: reference minigpt4.cpp:2897-2935).  Values follow
// ggml's dequantize_row_q4_0 / q4_1 / q5_0 / q5_1 / q8_0 in F32 and are then rounded to F16 (RNE).
__device__ __forceinline__ float h16_at(const unsigned char *p) { return __half2float(__ushort_as_half((unsigned short)(p[0] | (p[1] << 8)))); }
__global__ void dequant_to_f16_kernel(int gg_type, const unsigned char *__restrict__ raw, size_t n, __half *__restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const size_t b = i >> 5; const int j = (int)(i & 31), jj = j & 15;
    float v = 0.f;
    switch (gg_type) {
        case GG_F32: v = ((const float *)raw)[i]; break;
        case GG_Q4_0: { const unsigned char *p = raw + b * 18; const int q = j < 16 ? (p[2 + jj] & 0xF) : (p[2 + jj] >> 4); v = (float)(q - 8) * h16_at(p); break; }
        case GG_Q4_1: { const unsigned char *p = raw + b * 20; const int q = j < 16 ? (p[4 + jj] & 0xF) : (p[4 + jj] >> 4); v = (float)q * h16_at(p) + h16_at(p + 2); break; }
        case GG_Q5_0: { const unsigned char *p = raw + b * 22; const unsigned qh = p[2] | (p[3] << 8) | (p[4] << 16) | ((unsigned)p[5] << 24);
            const int q = (j < 16 ? (p[6 + jj] & 0xF) : (p[6 + jj] >> 4)) | (int)(((qh >> j) & 1u) << 4); v = (float)(q - 16) * h16_at(p); break; }
        case GG_Q5_1: { const unsigned char *p = raw + b * 24; const unsigned qh = p[4] | (p[5] << 8) | (p[6] << 16) | ((unsigned)p[7] << 24);
            const int q = (j < 16 ? (p[8 + jj] & 0xF) : (p[8 + jj] >> 4)) | (int)(((qh >> j) & 1u) << 4); v = (float)q * h16_at(p) + h16_at(p + 2); break; }
        case GG_Q8_0: { const unsigned char *p = raw + b * 34; v = (float)(signed char)p[2 + j] * h16_at(p); break; }
    }
    out[i] = __float2half_rn(v);
}

}  // namespace vk
}  // namespace mg4

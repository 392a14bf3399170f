// llama_sample.cuh — sm_90a kernels of the device sampler (minigpt4_b200_sample_steps; host side LlamaDevice::sample_steps in llama.cu,
// DESIGN.md §4.9): the reference's non-mirostat chain (minigpt4.cpp:2472-2477: top_k -> tail_free -> typical -> top_p -> temperature ->
// draw) and its mirostat v1 / v2 branches (:2456-2468) restated operation for operation from the host Sampler (text.cpp), so that a
// context draws the ids its host Sampler would draw from the same mt19937 state, and leaves the same mirostat μ.
//
// One CTA per context.  Element-wise work is spread over the CTA; every float sum the host takes sequentially (softmax, tail_free's
// accumulate, the entropy, the cumulative cuts, the double sums of std::discrete_distribution) is taken by thread 0 in candidate order.
// The build passes -fmad=false, so nothing is contracted except the fma() calls written out in the libm twins below.
//
// The one way the device can differ from the host: candidates with EQUAL sort keys (equal logits in the top-k / softmax sort, equal
// |-log p - H| in typical's sort) are ordered by lower id (lower index) here, while libstdc++'s heap / introsort leaves them in an
// order of its own.  Equal values give equal float results, so a tie can only change which of the tied ids is returned.
#pragma once
#include "llama.h"

namespace mg4 {
namespace smp {

constexpr int kThreads = 1024;
constexpr int kSmemSort = 4096;   // sorts of up to this many keys run in shared memory, larger ones in the context's scratch
constexpr int kMtN = 624, kMtM = 397;

// ---------------------------------------------------------------------------------------------------------------------------------
// glibc's expf / logf (the ARM optimized-routines algorithms glibc ships, as its x86-64 FMA variants evaluate them), bit for bit.
// CUDA's expf / logf round differently; the host Sampler calls glibc's.
// ---------------------------------------------------------------------------------------------------------------------------------
__constant__ unsigned long long kExp2fTab[32] = {   // asuint64(2^(i/32)) - (i << 47)
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull, 0x3fef72b83c7d517bull, 0x3fef54873168b9aaull,
    0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull, 0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull, 0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull,
    0x3feea11473eb0187ull, 0x3feea589994cce13ull, 0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull, 0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full,
    0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};
__constant__ double kLogfTab[16][2] = {   // {1/c, log c} of the 16 subintervals
    {0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2}, {0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2}, {0x1.49539f0f010bp+0, -0x1.01eae7f513a67p-2},
    {0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3}, {0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3}, {0x1.25e227b0b8eap+0, -0x1.1aa2bc79c81p-3},
    {0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4}, {0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4}, {0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5},
    {0x1p+0, 0x0p+0}, {0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5}, {0x1.ca4b31f026aap-1, 0x1.c5e53aa362eb4p-4},
    {0x1.b2036576afce6p-1, 0x1.526e57720db08p-3}, {0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3}, {0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2},
    {0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2}};

__device__ __forceinline__ float glibc_expf(float x) {
    const unsigned ux = __float_as_uint(x), abstop = (ux >> 20) & 0x7ff;
    if (abstop >= 0x42b) {   // |x| >= 88 or not finite
        if (ux == 0xff800000u) return 0.0f;
        if (abstop >= 0x7f8) return x + x;
        if (x > 0x1.62e42ep6f) return __int_as_float(0x7f800000);
        if (x < -0x1.9fe368p6f) return 0.0f;
    }
    const double inv_ln2_n = 0x1.71547652b82fep+0 * 32, shift = 0x1.8p+52;
    const double c0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, c1 = 0x1.ebfce50fac4f3p-3 / 32 / 32, c2 = 0x1.62e42ff0c52d6p-1 / 32;
    const double xd = (double)x;
    double kd = __fma_rn(inv_ln2_n, xd, shift);   // x N / ln2 = k + r, rounded to nearest through the shift
    const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
    kd = __dsub_rn(kd, shift);
    const double r = __fma_rn(inv_ln2_n, xd, -kd);
    const unsigned long long t = kExp2fTab[ki % 32] + (ki << 47);
    const double s = __longlong_as_double((long long)t);
    const double z = __fma_rn(c0, r, c1), r2 = __dmul_rn(r, r);
    double y = __fma_rn(c2, r, 1.0);
    y = __fma_rn(z, r2, y);
    return __double2float_rn(__dmul_rn(y, s));
}

__device__ __forceinline__ float glibc_logf(float x) {
    unsigned ix = __float_as_uint(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {   // x < 0x1p-126, inf or nan
        if (ix * 2 == 0) return __int_as_float(0xff800000);
        if (ix == 0x7f800000u) return x;
        if ((ix & 0x80000000u) || ix * 2 >= 0xff000000u) return __int_as_float(0x7fc00000);
        ix = __float_as_uint(__fmul_rn(x, 0x1p23f));   // subnormal: normalise
        ix -= 23u << 23;
    }
    const double ln2 = 0x1.62e42fefa39efp-1, a0 = -0x1.00ea348b88334p-2, a1 = 0x1.5575b0be00b6ap-2, a2 = -0x1.ffffef20a4123p-2;
    const unsigned tmp = ix - 0x3f330000u;
    const int i = (int)((tmp >> 19) % 16), kx = (int)tmp >> 23;
    const unsigned iz = ix - (tmp & (0x1ffu << 23));
    const double invc = kLogfTab[i][0], logc = kLogfTab[i][1], z = (double)__uint_as_float(iz);
    const double r = __fma_rn(z, invc, -1.0);
    const double y0 = __fma_rn((double)kx, ln2, logc);
    const double r2 = __dmul_rn(r, r);
    double y = __fma_rn(a1, r, a2);
    y = __fma_rn(a0, r2, y);
    y = __fma_rn(y, r2, __dadd_rn(y0, r));
    return __double2float_rn(y);
}

// fn 0: expf, 1: logf of the float bit patterns lo .. lo + n - 1
__global__ void libm_kernel(int fn, unsigned lo, unsigned n, float *out) {
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float x = __uint_as_float(lo + i);
        out[i] = fn == 0 ? glibc_expf(x) : glibc_logf(x);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// glibc's log2f / powf for mirostat (same algorithms and FMA evaluation as above), bit for bit, NaN results included: where the host's
// result is a NaN, these give the NaN an x86-64 SSE operation gives (a NaN operand comes back quieted, the first one if both are; an
// invalid operation gives the default NaN 0xffc00000), while CUDA's float operations always give 0x7fffffff.
// ---------------------------------------------------------------------------------------------------------------------------------
__constant__ double kLog2fTab[16][2] = {   // {1/c, log2 c} of the 16 subintervals, shared by log2f and powf's log2
    {0x1.661ec79f8f3bep+0, -0x1.efec65b963019p-2}, {0x1.571ed4aaf883dp+0, -0x1.b0b6832d4fca4p-2}, {0x1.49539f0f010bp+0, -0x1.7418b0a1fb77bp-2},
    {0x1.3c995b0b80385p+0, -0x1.39de91a6dcf7bp-2}, {0x1.30d190c8864a5p+0, -0x1.01d9bf3f2b631p-2}, {0x1.25e227b0b8eap+0, -0x1.97c1d1b3b7afp-3},
    {0x1.1bb4a4a1a343fp+0, -0x1.2f9e393af3c9fp-3}, {0x1.12358f08ae5bap+0, -0x1.960cbbf788d5cp-4}, {0x1.0953f419900a7p+0, -0x1.a6f9db6475fcep-5},
    {0x1p+0, 0x0p+0}, {0x1.e608cfd9a47acp-1, 0x1.338ca9f24f53dp-4}, {0x1.ca4b31f026aap-1, 0x1.476a9543891bap-3},
    {0x1.b2036576afce6p-1, 0x1.e840b4ac4e4d2p-3}, {0x1.9c2d163a1aa2dp-1, 0x1.40645f0c6651cp-2}, {0x1.886e6037841edp-1, 0x1.88e9c2c1b9ff8p-2},
    {0x1.767dcf5534862p-1, 0x1.ce0a44eb17bccp-2}};

// the NaN an x86 operation on a and b returns when its result is a NaN
__device__ __forceinline__ float x86_nan(float a, float b) {
    if (isnan(a)) return __uint_as_float(__float_as_uint(a) | 0x00400000u);
    if (isnan(b)) return __uint_as_float(__float_as_uint(b) | 0x00400000u);
    return __uint_as_float(0xffc00000u);
}
__device__ __forceinline__ float neg(float x) { return __uint_as_float(__float_as_uint(x) ^ 0x80000000u); }   // x86's -x: the sign bit, NaN too

__device__ __forceinline__ float glibc_log2f(float x) {
    unsigned ix = __float_as_uint(x);
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {   // x < 0x1p-126, inf or nan
        if (ix * 2 == 0) return __int_as_float(0xff800000);
        if (ix == 0x7f800000u) return x;
        if ((ix & 0x80000000u) || ix * 2 >= 0xff000000u) return x86_nan(x, x);   // (x - x) / (x - x)
        ix = __float_as_uint(__fmul_rn(x, 0x1p23f));   // subnormal: normalise
        ix -= 23u << 23;
    }
    const double a0 = -0x1.712b6f70a7e4dp-2, a1 = 0x1.ecabf496832ep-2, a2 = -0x1.715479ffae3dep-1, a3 = 0x1.715475f35c8b8p0;
    const unsigned tmp = ix - 0x3f330000u;
    const int i = (int)((tmp >> 19) % 16), k = (int)tmp >> 23;
    const unsigned iz = ix - (tmp & 0xff800000u);
    const double invc = kLog2fTab[i][0], logc = kLog2fTab[i][1], z = (double)__uint_as_float(iz);
    const double r = __fma_rn(z, invc, -1.0);
    const double y0 = __dadd_rn(logc, (double)k);
    const double r2 = __dmul_rn(r, r);
    double y = __fma_rn(a1, r, a2);
    y = __fma_rn(a0, r2, y);
    y = __fma_rn(y, r2, __fma_rn(a3, r, y0));
    return __double2float_rn(y);
}

// powf's test of a finite non-zero y: 0 not an integer, 1 odd, 2 even
__device__ __forceinline__ int powf_checkint(unsigned iy) {
    const int e = iy >> 23 & 0xff;
    if (e < 0x7f) return 0;
    if (e > 0x7f + 23) return 2;
    if (iy & ((1u << (0x7f + 23 - e)) - 1)) return 0;
    if (iy & (1u << (0x7f + 23 - e))) return 1;
    return 2;
}
__device__ __forceinline__ bool powf_zeroinfnan(unsigned ix) { return 2 * ix - 1 >= 2u * 0x7f800000u - 1; }

__device__ __forceinline__ float glibc_powf(float x, float y) {
    unsigned sign_bias = 0, ix = __float_as_uint(x);
    const unsigned iy = __float_as_uint(y);
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u || powf_zeroinfnan(iy)) {   // x < 0x1p-126, inf or nan; or y 0, inf or nan
        if (powf_zeroinfnan(iy)) {
            if (2 * iy == 0) return isnan(x) && !(ix & 0x00400000u) ? x86_nan(x, y) : 1.0f;   // (signalling x: x + y)
            if (ix == 0x3f800000u) return isnan(y) && !(iy & 0x00400000u) ? x86_nan(x, y) : 1.0f;
            if (2 * ix > 2u * 0x7f800000u || 2 * iy > 2u * 0x7f800000u) return x86_nan(x, y);
            if (2 * ix == 2 * 0x3f800000u) return 1.0f;
            if ((2 * ix < 2 * 0x3f800000u) == !(iy & 0x80000000u)) return 0.0f;   // |x| < 1 and y inf, or |x| > 1 and y -inf
            return __fmul_rn(y, y);
        }
        if (powf_zeroinfnan(ix)) {
            float x2 = isnan(x) ? x86_nan(x, x) : __fmul_rn(x, x);
            if ((ix & 0x80000000u) && powf_checkint(iy) == 1) x2 = neg(x2);
            if (iy & 0x80000000u) return isnan(x2) ? x86_nan(x2, x2) : __fdiv_rn(1.0f, x2);
            return x2;
        }
        if (ix & 0x80000000u) {   // finite x < 0
            const int yint = powf_checkint(iy);
            if (yint == 0) return __uint_as_float(0xffc00000u);
            if (yint == 1) sign_bias = 1u << 16;
            ix &= 0x7fffffffu;
        }
        if (ix < 0x00800000u) {   // subnormal x: normalise (the exponent goes negative)
            ix = __float_as_uint(__fmul_rn(x, 0x1p23f));
            ix &= 0x7fffffffu;
            ix -= 23u << 23;
        }
    }
    // log2(x) in double
    const double a0 = 0x1.27616c9496e0bp-2, a1 = -0x1.71969a075c67ap-2, a2 = 0x1.ec70a6ca7baddp-2, a3 = -0x1.7154748bef6c8p-1,
                 a4 = 0x1.71547652ab82bp+0;
    const unsigned tmp = ix - 0x3f330000u, top = tmp & 0xff800000u;
    const int i = (int)((tmp >> 19) % 16), k = (int)top >> 23;
    const double invc = kLog2fTab[i][0], logc = kLog2fTab[i][1], z = (double)__uint_as_float(ix - top);
    const double r = __fma_rn(z, invc, -1.0), y0 = __dadd_rn(logc, (double)k), r2 = __dmul_rn(r, r);
    double l = __fma_rn(a0, r, a1);
    const double p = __fma_rn(a2, r, a3), r4 = __dmul_rn(r2, r2);
    double q = __fma_rn(a4, r, y0);
    q = __fma_rn(p, r2, q);
    l = __fma_rn(l, r4, q);
    const double ylogx = __dmul_rn((double)y, l);
    if (((unsigned long long)__double_as_longlong(ylogx) >> 47 & 0xffff) >= 0x80bfu) {   // |y log2 x| >= 126 (asuint64(126.0) >> 47)
        if (ylogx > 0x1.fffffffd1d571p+6) return sign_bias ? __int_as_float(0xff800000) : __int_as_float(0x7f800000);   // overflow
        if (ylogx <= -150.0) return sign_bias ? -0.0f : 0.0f;                                                             // underflow
    }
    // 2^ylogx as expf's exp2 (kExp2fTab), the sign from sign_bias
    const double shift = 0x1.8p+52 / 32, c0 = 0x1.c6af84b912394p-5, c1 = 0x1.ebfce50fac4f3p-3, c2 = 0x1.62e42ff0c52d6p-1;
    double kd = __dadd_rn(ylogx, shift);
    const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
    kd = __dsub_rn(kd, shift);
    const double rr = __dsub_rn(ylogx, kd);
    const unsigned long long t = kExp2fTab[ki % 32] + ((ki + sign_bias) << 47);
    const double s = __longlong_as_double((long long)t);
    const double zz = __fma_rn(c0, rr, c1), rr2 = __dmul_rn(rr, rr);
    double w = __fma_rn(c2, rr, 1.0);
    w = __fma_rn(zz, rr2, w);
    return __double2float_rn(__dmul_rn(w, s));
}

// (int)f as x86-64's cvttss2si computes it: truncation, and INT_MIN for NaN and for anything outside the int range
__device__ __forceinline__ int x86_cvtt(float f) {
    return f >= -2147483648.0f && f < 2147483648.0f ? __float2int_rz(f) : (int)0x80000000u;
}

// fn 0: log2f of the float bit patterns lo .. lo + n - 1; fn 1: powf(x, y) for the y of those bit patterns
__global__ void mirostat_libm_kernel(int fn, float x, unsigned lo, unsigned n, float *out) {
    for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float v = __uint_as_float(lo + i);
        out[i] = fn == 0 ? glibc_log2f(v) : glibc_powf(x, v);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// the sampler
// ---------------------------------------------------------------------------------------------------------------------------------
struct MtState { unsigned x[kMtN]; unsigned p; };   // std::mt19937's state: 624 words and the position in them

// one context's column of a sampling launch; the scratch pointers are its SamplerScratch (LlamaDevice::ensure_sampler)
struct SampleCtx {
    const float *logits;
    DeviceState *state;          // tokens[0] takes the sampled id, which the decode step then feeds
    SessionSlot *slot;           // batched steps: the context's column, whose position is n_past0 + step
    int n_past0;
    MtState *mt;
    int *ids;                    // [n_ctx] the id fed at each step of a call
    unsigned long long *keys;    // [pow2 >= n_vocab] sort keys; the discrete distribution's cumulative doubles afterwards
    int *id; float *logit, *p, *aux;   // [n_vocab] candidates (id, logit, probability); tail_free's d2 / typical's terms
    SamplingArgs args;           // the column's sampling parameters (mirostat 1 / 2: the mirostat kernels, which ignore top_k .. typical_p)
};
// a sampling launch's arguments, one column per CTA; the table is passed by value, so its capacity N is part of the kernel's parameters:
// N = 8 for launches of 1..8 contexts, kMaxBatch for wider ones
template <int N> struct SampleArgsN {
    SampleCtx c[N];
    int n_vocab, step;
};

// float -> key that orders like the float (-0 as +0, so that equal logits are equal keys), and back
__device__ __forceinline__ unsigned ord_key(float v) {
    const unsigned u = __float_as_uint(v == 0.0f ? 0.0f : v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ord_val(unsigned o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }
// descending order of these keys = logit descending, ties by lower id
__device__ __forceinline__ unsigned long long desc_key(float v, int id) { return ((unsigned long long)ord_key(v) << 32) | (0xFFFFFFFFu - (unsigned)id); }
__device__ __forceinline__ int key_id(unsigned long long k) { return (int)(0xFFFFFFFFu - (unsigned)(k & 0xFFFFFFFFull)); }

__device__ __forceinline__ int pow2_at_least(int n) { int P = 2; while (P < n) P <<= 1; return P; }

// one bitonic compare-exchange pass of stride st over buf[0, n) whose element 0 is element base of the whole sequence (the direction of
// a pair follows its position in the whole sequence: descending where (position & size) == 0)
__device__ __forceinline__ void bitonic_pass(unsigned long long *buf, int n, int base, int size, int st) {
    for (int i = threadIdx.x; i < n / 2; i += blockDim.x) {
        const int lo = 2 * i - (i & (st - 1)), hi = lo + st;
        const bool desc = ((base + lo) & size) == 0;
        const unsigned long long a = buf[lo], b = buf[hi];
        if ((a < b) == desc) { buf[lo] = b; buf[hi] = a; }
    }
    __syncthreads();
}

// bitonic sort of buf[0, P) (P a power of two >= 2), descending.  Up to kSmemSort keys buf is sbuf itself; larger sequences live in
// global scratch, and every run of passes with strides below kSmemSort is done chunk by chunk in sbuf, so only the strides of
// kSmemSort and above make passes over global memory.
__device__ void bitonic_desc(unsigned long long *buf, int P, unsigned long long *sbuf) {
    constexpr int C = kSmemSort;
    if (P <= C) {
        for (int size = 2; size <= P; size <<= 1)
            for (int st = size >> 1; st > 0; st >>= 1) bitonic_pass(buf, P, 0, size, st);
        return;
    }
    auto local = [&](int size, int st0, bool all_sizes) {   // strides st0 .. 1 of every chunk (all_sizes: every size up to C first)
        for (int base = 0; base < P; base += C) {
            for (int i = threadIdx.x; i < C; i += blockDim.x) sbuf[i] = buf[base + i];
            __syncthreads();
            if (all_sizes) {
                for (int sz = 2; sz <= C; sz <<= 1)
                    for (int st = sz >> 1; st > 0; st >>= 1) bitonic_pass(sbuf, C, base, sz, st);
            } else {
                for (int st = st0; st > 0; st >>= 1) bitonic_pass(sbuf, C, base, size, st);
            }
            for (int i = threadIdx.x; i < C; i += blockDim.x) buf[base + i] = sbuf[i];
            __syncthreads();
        }
    };
    local(0, 0, true);
    for (int size = 2 * C; size <= P; size <<= 1) {
        int st = size >> 1;
        for (; st >= C; st >>= 1) bitonic_pass(buf, P, 0, size, st);
        local(size, st, false);
    }
}

// the n candidates sorted by logit, descending (Sampler's by_logit_desc), ties by lower id; p is recomputed by the softmax that follows
__device__ void sort_by_logit(const SampleCtx &c, int n, unsigned long long *sbuf) {
    const int P = pow2_at_least(n);
    unsigned long long *buf = P <= kSmemSort ? sbuf : c.keys;
    for (int i = threadIdx.x; i < P; i += blockDim.x) buf[i] = i < n ? desc_key(c.logit[i], c.id[i]) : 0ull;
    __syncthreads();
    bitonic_desc(buf, P, sbuf);
    for (int i = threadIdx.x; i < n; i += blockDim.x) { c.id[i] = key_id(buf[i]); c.logit[i] = ord_val((unsigned)(buf[i] >> 32)); }
    __syncthreads();
}

// thread 0's in-order walk over x[0, n) for the sequential sums and cuts: 16 loads are issued before the 16 steps that use them, so their
// latencies overlap; the steps themselves run one after another in index order.  f(i, x[i]) returns false to stop.
template <class F> __device__ __forceinline__ void walk(const float *x, int n, F f) {
    int i = 0;
    for (; i + 16 <= n; i += 16) {
        float v[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = x[i + j];
#pragma unroll
        for (int j = 0; j < 16; ++j) if (!f(i + j, v[j])) return;
    }
    for (; i < n; ++i) if (!f(i, x[i])) return;
}

// Sampler::softmax over sorted candidates: p = expf(logit - max), summed in order, p /= sum
__device__ void softmax_sorted(const SampleCtx &c, int n, float *red) {
    const float mx = c.logit[0];
    for (int i = threadIdx.x; i < n; i += blockDim.x) c.p[i] = glibc_expf(c.logit[i] - mx);
    __syncthreads();
    if (threadIdx.x == 0) {
        float sum = 0.f;
        walk(c.p, n, [&](int, float v) { sum += v; return true; });
        *red = sum;
    }
    __syncthreads();
    const float sum = *red;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c.p[i] = c.p[i] / sum;
    __syncthreads();
}

// std::mt19937's next output, as libstdc++ produces it: all 624 words are regenerated when the position reaches the end
__device__ unsigned mt_next(MtState &m) {
    if (m.p >= (unsigned)kMtN) {
        const unsigned upper = 0x80000000u, lower = 0x7fffffffu, a = 0x9908b0dfu;
        int k = 0;
        for (; k < kMtN - kMtM; ++k) { const unsigned y = (m.x[k] & upper) | (m.x[k + 1] & lower); m.x[k] = m.x[k + kMtM] ^ (y >> 1) ^ ((y & 1u) ? a : 0u); }
        for (; k < kMtN - 1; ++k) { const unsigned y = (m.x[k] & upper) | (m.x[k + 1] & lower); m.x[k] = m.x[k + kMtM - kMtN] ^ (y >> 1) ^ ((y & 1u) ? a : 0u); }
        const unsigned y = (m.x[kMtN - 1] & upper) | (m.x[0] & lower);
        m.x[kMtN - 1] = m.x[kMtM - 1] ^ (y >> 1) ^ ((y & 1u) ? a : 0u);
        m.p = 0;
    }
    unsigned z = m.x[m.p++];
    z ^= z >> 11;
    z ^= (z << 7) & 0x9d2c5680u;
    z ^= (z << 15) & 0xefc60000u;
    z ^= z >> 18;
    return z;
}

// thread 0's draw over the m candidates whose probabilities softmax_sorted left in c.p: std::discrete_distribution<int> over the float
// probabilities, as Sampler::draw; hands the drawn index to drawn(idx)
template <class Drawn> __device__ __forceinline__ void draw(const SampleCtx &c, int m, MtState &mt, Drawn drawn) {
    int idx = 0;   // one candidate: index 0, no draw from the generator
    if (m >= 2) {
        double sum = 0.0;
        walk(c.p, m, [&](int, float v) { sum += (double)v; return true; });
        double *cp = (double *)c.keys, acc = 0.0;
        walk(c.p, m, [&](int i, float v) { acc += (double)v / sum; cp[i] = acc; return true; });
        cp[m - 1] = 1.0;
        // generate_canonical<double, 53>: two 32-bit outputs, (a + b 2^32) / 2^64, kept below 1
        const double lo = (double)mt_next(mt), hi = (double)mt_next(mt);
        double u = (lo + hi * 4294967296.0) / 18446744073709551616.0;
        if (u >= 1.0) u = 0x1.fffffffffffffp-1;
        int first = 0, len = m;   // std::lower_bound
        while (len > 0) {
            const int half = len >> 1, mid = first + half;
            if (cp[mid] < u) { first = mid + 1; len = len - half - 1; }
            else len = half;
        }
        idx = first;
    }
    drawn(idx);
}

// the candidates of a sampling step, in the order the host Sampler lists them: every id of the vocabulary, or a constrained column's
// allowed ids, ascending (its state's row of the constraint table, constraint.h).  sample_body takes them from its argument type
// (cand_*), so the kernels that sample every id instantiate it exactly as before.
struct AllowedIds {
    const int2 *tr;   // the row's (id, next state) pairs; null: an unconstrained column of a constrained launch, every id
    int n;
    __device__ __forceinline__ bool listed() const { return tr != nullptr; }
};
// a constrained launch's column: its candidates
struct ListedArgs {
    int n_vocab;
    AllowedIds src;
};
template <class A> struct CandTraits { static constexpr bool kListed = false; };
template <> struct CandTraits<ListedArgs> { static constexpr bool kListed = true; };
template <class A> __device__ __forceinline__ int cand_size(const A &a) { return a.n_vocab; }
template <class A> __device__ __forceinline__ int cand_id(const A &, int j) { return j; }
template <class A> __device__ __forceinline__ bool cand_listed(const A &) { return false; }
__device__ __forceinline__ int cand_size(const ListedArgs &a) { return a.src.n; }
__device__ __forceinline__ int cand_id(const ListedArgs &a, int j) { return a.src.tr ? a.src.tr[j].x : j; }
__device__ __forceinline__ bool cand_listed(const ListedArgs &a) { return a.src.listed(); }

// ---------------------------------------------------------------------------------------------------------------------------------
// one context's sampling step, the body of sample_kernel and sample_cons_kernel (a CTA of kThreads): samples c's logits over the
// candidates of a (cand_*) as Sampler::sample (Sampler::sample_allowed for listed candidates) does with the column's parameters c.args,
// and hands the id to fed(id, greedy) on thread 0.  temp <= 0: the greedy id the logits epilogue already left in tokens[0] (greedy =
// true; the generator is not read), or for listed candidates their arg-max, the lower id on ties (greedy = false).  Otherwise the
// generator is written back after fed returns.
// ---------------------------------------------------------------------------------------------------------------------------------
template <class A, class Fed> __device__ __forceinline__ void sample_body(const A &a, const SampleCtx &c, Fed fed) {
    __shared__ unsigned long long sbuf[kSmemSort];
    __shared__ MtState mt;
    __shared__ unsigned hist[256];
    __shared__ unsigned long long sh_prefix;
    __shared__ int sh_need, sh_done, sh_n;
    __shared__ float red;
    const int tid = threadIdx.x, n = cand_size(a);
    if (c.args.temp <= 0.f) {
        if constexpr (CandTraits<A>::kListed) {
            if (cand_listed(a)) {
                if (tid == 0) sh_prefix = 0ull;
                __syncthreads();
                unsigned long long best = 0ull;
                for (int j = tid; j < n; j += blockDim.x) { const int i = cand_id(a, j); best = max(best, desc_key(c.logits[i], i)); }
                atomicMax(&sh_prefix, best);
                __syncthreads();
                if (tid == 0) fed(key_id(sh_prefix), false);
                return;
            }
        }
        if (tid == 0) fed(c.state->tokens[0], true);
        return;
    }
    for (int i = tid; i < kMtN; i += blockDim.x) mt.x[i] = c.mt->x[i];
    if (tid == 0) mt.p = c.mt->p;

    // ---- top_k: the k largest (logit desc, id asc) keys; k = top_k (<= 0: all candidates) clamped to [1, candidates] as Sampler::top_k does
    const int k = min(max(c.args.top_k <= 0 ? n : c.args.top_k, 1), n);
    if (k == n) {
        if constexpr (CandTraits<A>::kListed) {
            for (int j = tid; j < n; j += blockDim.x) { const int i = cand_id(a, j); c.id[j] = i; c.logit[j] = c.logits[i]; }
        } else {   // (written as before: the every-id kernels compile to the same code)
            for (int i = tid; i < n; i += blockDim.x) { c.id[i] = i; c.logit[i] = c.logits[i]; }
        }
    } else {
        // radix select, 8 bits at a time from the top: the threshold T with exactly k keys >= T (keys are distinct: they carry the id)
        unsigned long long mask = 0ull;
        if (tid == 0) { sh_prefix = 0ull; sh_need = k; }
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0u;
            __syncthreads();
            const unsigned long long pre = sh_prefix;
            for (int i = tid; i < n; i += blockDim.x) {
                const unsigned long long key = desc_key(c.logits[cand_id(a, i)], cand_id(a, i));
                if ((key & mask) == pre) atomicAdd(&hist[(key >> shift) & 255], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                int need = sh_need, d = 255; unsigned cum = 0;
                for (; d > 0; --d) { if (cum + hist[d] >= (unsigned)need) break; cum += hist[d]; }
                need -= (int)cum;
                sh_prefix = pre | ((unsigned long long)d << shift);
                sh_need = need;
                sh_done = hist[d] == (unsigned)need;   // every key of this prefix is in: T = the prefix
            }
            __syncthreads();
            mask |= 255ull << shift;
            if (sh_done) break;
        }
        if (tid == 0) sh_n = 0;
        __syncthreads();
        const unsigned long long T = sh_prefix;
        for (int i = tid; i < n; i += blockDim.x) {
            const float v = c.logits[cand_id(a, i)];
            if (desc_key(v, cand_id(a, i)) >= T) { const int j = atomicAdd(&sh_n, 1); c.id[j] = cand_id(a, i); c.logit[j] = v; }
        }
    }
    __syncthreads();
    sort_by_logit(c, k, sbuf);
    int m = k;
    bool sorted = true;

    // ---- tail_free
    if (c.args.tfs_z < 1.0f && m > 2) {
        softmax_sorted(c, m, &red);
        for (int i = tid; i < m - 2; i += blockDim.x) {
            const float d1a = c.p[i] - c.p[i + 1], d1b = c.p[i + 1] - c.p[i + 2];
            c.aux[i] = fabsf(d1a - d1b);
        }
        __syncthreads();
        if (tid == 0) {
            float s = 0.f;
            walk(c.aux, m - 2, [&](int, float v) { s += v; return true; });
            float cum = 0.f; int last = m;
            walk(c.aux, m - 2, [&](int i, float v) { cum += v / s; if (cum > c.args.tfs_z && i >= 1) { last = i; return false; } return true; });
            sh_n = last;
        }
        __syncthreads();
        m = sh_n;
    }

    // ---- typical: the candidates in order of |-log p - H| (ties by index) until their mass exceeds typical_p; leaves them unsorted
    if (c.args.typical_p < 1.0f) {
        softmax_sorted(c, m, &red);
        for (int i = tid; i < m; i += blockDim.x) c.aux[i] = -c.p[i] * glibc_logf(c.p[i]);
        __syncthreads();
        if (tid == 0) {
            float entropy = 0.f;
            walk(c.aux, m, [&](int, float v) { entropy += v; return true; });
            red = entropy;
        }
        __syncthreads();
        const float entropy = red;
        const int P = pow2_at_least(m);
        unsigned long long *buf = P <= kSmemSort ? sbuf : c.keys;
        for (int i = tid; i < P; i += blockDim.x) {   // descending order of ~shifted = ascending shifted, ties by lower index
            if (i < m) {
                const float shifted = fabsf(-glibc_logf(c.p[i]) - entropy);
                buf[i] = ((unsigned long long)(~ord_key(shifted)) << 32) | (0xFFFFFFFFu - (unsigned)i);
            } else buf[i] = 0ull;
        }
        __syncthreads();
        bitonic_desc(buf, P, sbuf);
        if (tid == 0) {
            float cum = 0.f; int last = m;
            for (int i = 0; i < m; ++i) { cum += c.p[key_id(buf[i])]; if (cum > c.args.typical_p) { last = i + 1; break; } }
            sh_n = last;
        }
        __syncthreads();
        const int last = sh_n;
        for (int i = tid; i < last; i += blockDim.x) {   // gather the kept candidates in that order (through buf: in place)
            const int j = key_id(buf[i]);
            buf[i] = ((unsigned long long)(unsigned)c.id[j] << 32) | __float_as_uint(c.logit[j]);
        }
        __syncthreads();
        for (int i = tid; i < last; i += blockDim.x) { c.id[i] = (int)(buf[i] >> 32); c.logit[i] = __uint_as_float((unsigned)buf[i]); }
        __syncthreads();
        m = last;
        sorted = false;
    }

    // ---- top_p
    if (c.args.top_p < 1.0f) {
        if (!sorted) { sort_by_logit(c, m, sbuf); sorted = true; }
        softmax_sorted(c, m, &red);
        if (tid == 0) {
            float cum = 0.f; int last = m;
            walk(c.p, m, [&](int i, float v) { cum += v; if (cum >= c.args.top_p) { last = i + 1; return false; } return true; });
            sh_n = last;
        }
        __syncthreads();
        m = sh_n;
    }

    // ---- temperature, then draw: softmax, std::discrete_distribution<int> over the float probabilities
    for (int i = tid; i < m; i += blockDim.x) c.logit[i] = c.logit[i] / c.args.temp;
    __syncthreads();
    if (!sorted) sort_by_logit(c, m, sbuf);
    softmax_sorted(c, m, &red);
    if (tid == 0) draw(c, m, mt, [&](int idx) { fed(c.id[idx], false); });
    __syncthreads();
    for (int i = tid; i < kMtN; i += blockDim.x) c.mt->x[i] = mt.x[i];
    if (tid == 0) c.mt->p = mt.p;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// one context's mirostat step, the body of sample_kernel<N, true>: Sampler::sample's mirostat branch
// (c.args.mirostat 1 or 2, its tau and eta) with its μ in `ms`, handing the id to fed(id, greedy) on thread 0.  temp <= 0: the greedy
// id, and neither μ nor the generator is read.  Otherwise μ is set to 2 tau at the mode's first use, as on the host, and updated after
// the draw.
// ---------------------------------------------------------------------------------------------------------------------------------
// a context's μ: right after its generator in its SamplerScratch (llama.cu), so that one copy moves both
__device__ __forceinline__ MirostatState &mirostat_state(const SampleCtx &c) { return *(MirostatState *)(c.mt + 1); }

template <class A, class Fed>
__device__ __forceinline__ void mirostat_body(const A &a, const SampleCtx &c, MirostatState &ms, Fed fed) {
    __shared__ unsigned long long sbuf[kSmemSort];
    __shared__ MtState mt;
    __shared__ int sh_n;
    __shared__ float red;
    const SamplingArgs &ma = c.args;
    const int tid = threadIdx.x, n = a.n_vocab, v = ma.mirostat - 1;
    if (ma.temp <= 0.f) {
        if (tid == 0) fed(c.state->tokens[0], true);
        return;
    }
    for (int i = tid; i < kMtN; i += blockDim.x) mt.x[i] = c.mt->x[i];
    if (tid == 0) {
        mt.p = c.mt->p;
        if (!ms.init[v]) { ms.mu[v] = 2.0f * ma.mirostat_tau; ms.init[v] = 1; }
        sh_n = n;
    }
    // temperature over the whole vocabulary, then the sort by the divided logit and the softmax
    for (int i = tid; i < n; i += blockDim.x) { c.id[i] = i; c.logit[i] = c.logits[i] / ma.temp; }
    __syncthreads();
    sort_by_logit(c, n, sbuf);
    softmax_sorted(c, n, &red);
    const float mu = ms.mu[v];
    if (v == 0) {
        // v1: Zipf exponent from the first 100 probabilities (in order, on one thread), then k from it and μ; top_k(k, 1)
        if (tid == 0) {
            float s_tb = 0.f, s_tt = 0.f;
            for (int i = 0; i < 99 && i + 1 < n; ++i) {
                const float t = glibc_logf((float)(i + 2) / (float)(i + 1)), b = glibc_logf(c.p[i] / c.p[i + 1]);
                s_tb += t * b; s_tt += t * t;
            }
            const float s_hat = s_tb / s_tt, eps = s_hat - 1;
            const float kf = glibc_powf((eps * glibc_powf(2.0f, mu)) / (1 - glibc_powf((float)n, -eps)), 1 / s_hat);
            sh_n = min(max(x86_cvtt(kf), 1), n);
        }
    } else {
        // v2: the leading candidates of surprise -log2 p <= μ, at least one (the first that fails ends the host's loop)
        for (int i = tid; i < n; i += blockDim.x)
            if (!(-glibc_log2f(c.p[i]) <= mu)) atomicMin(&sh_n, max(i, 1));
    }
    __syncthreads();
    const int m = sh_n;
    softmax_sorted(c, m, &red);
    if (tid == 0) draw(c, m, mt, [&](int idx) {
        fed(c.id[idx], false);
        // μ -= eta (surprise - tau) with the drawn candidate's probability after the draw's softmax, NaNs as on x86
        const float s = neg(glibc_log2f(c.p[idx]));
        float d = s - ma.mirostat_tau;
        if (isnan(d)) d = x86_nan(s, ma.mirostat_tau);
        float e = ma.mirostat_eta * d;
        if (isnan(e)) e = x86_nan(ma.mirostat_eta, d);
        float r = mu - e;
        if (isnan(r)) r = x86_nan(mu, e);
        ms.mu[v] = r;
    });
    __syncthreads();
    for (int i = tid; i < kMtN; i += blockDim.x) c.mt->x[i] = mt.x[i];
    if (tid == 0) c.mt->p = mt.p;
}

// the id a step feeds: into tokens[0] (the greedy id is already there) and ids[step]; a batched column moves to its next position
template <class A> __device__ __forceinline__ void feed(const A &a, const SampleCtx &c, int id, bool greedy) {
    if (!greedy) c.state->tokens[0] = id;
    c.ids[a.step] = id;
    if (c.slot) c.slot->n_past = c.n_past0 + a.step;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// stop on the reply's text (minigpt4_b200_sample_until; host side LlamaDevice::sample_until): the reference's chat loop
// (MiniGPT4ChatBot.generate) appends each token's text to the reply and stops after a token that is not exactly "##" once the reply
// ends with "###".  The text of an id is the C string of Engine::id_to_token, from the group's token table.
// ---------------------------------------------------------------------------------------------------------------------------------
constexpr int kStopMax = LlamaDevice::kStopMax;   // longest stop text; the reply's last kStopMax bytes decide every later check

struct TokenTable { const int *off; const unsigned char *bytes; };   // id's text: bytes[off[id], off[id + 1])

struct ReplyState {                  // one context's stop state in a call (the host writes it before the first step)
    unsigned char tail[kStopMax];    // the reply's last tail_len bytes
    unsigned char stop[kStopMax];
    int tail_len, stop_len;          // stop_len 0: no text stop
    int done;                        // 0 running; 1 stopped at the previous step; 2 stopped, logits and state in the snapshot
    int n_fed;                       // steps that fed an id
    DeviceState snap;
};
struct UntilState : ReplyState {     // a context's state in a sample_until call (beam search keeps bare ReplyStates)
    int budget;                      // the context's max_steps: it is done once n_fed reaches it
    int by_budget;                   // 1: the budget, not the text (or </s>), ended it
};

// the reply takes id's text; returns true if that step ends it.  One thread; no local arrays.
__device__ __forceinline__ bool reply_take(ReplyState &r, TokenTable t, int id) {
    const unsigned char *piece = t.bytes + t.off[id];
    const int len = t.off[id + 1] - t.off[id], tl = r.tail_len;
    bool stop = r.stop_len > 0 && !(len == 2 && piece[0] == '#' && piece[1] == '#') && tl + len >= r.stop_len;
    for (int k = 0; stop && k < r.stop_len; ++k) {   // byte k from the end of tail + piece
        const unsigned char b = k < len ? piece[len - 1 - k] : r.tail[tl - 1 - (k - len)];
        stop = b == r.stop[r.stop_len - 1 - k];
    }
    if (len >= kStopMax) {
        for (int k = 0; k < kStopMax; ++k) r.tail[k] = piece[len - kStopMax + k];
        r.tail_len = kStopMax;
    } else {
        const int keep = min(tl, kStopMax - len);
        for (int k = 0; k < keep; ++k) r.tail[k] = r.tail[tl - keep + k];
        for (int k = 0; k < len; ++k) r.tail[keep + k] = piece[k];
        r.tail_len = keep + len;
    }
    return stop;
}

template <int N> struct StopArgsN {
    UntilState *r[N];
    float *snap[N];   // [n_vocab] each context's logits after its last step
    TokenTable tab;
};
static_assert(sizeof(SampleArgsN<LlamaDevice::kMaxBatch>) + sizeof(StopArgsN<LlamaDevice::kMaxBatch>) <= 32764,
              "the widest kernel's parameters fit the 32 764-byte limit");

// one step of sample_kernel that stops each context on its reply's text or its budget.  A stopped context does not draw (its generator
// stays); at the next step it saves its logits and DeviceState, which the host restores at the end of the call.  The decode work that
// still runs for a batched column is parked: it feeds the column's last fed id again at that id's own position, so it rewrites the same
// K / V bits (the batched step is bit-exact per column) and never writes past the context's final n_past, which its budget keeps within
// n_ctx while other columns run on.
// the start of a step of the stopping kernels (sh_state: a __shared__ int of the kernel): false for a context that has stopped (it saves
// its snapshot once and parks its column), true for one that samples
template <class A, class S> __device__ __forceinline__ bool until_running(const A &a, const S &s, const SampleCtx &c, UntilState &r, int &sh_state) {
    if (threadIdx.x == 0) sh_state = r.done;   // (read once: thread 0 writes r.done when it feeds)
    __syncthreads();
    const int done = sh_state;
    if (done != 0) {
        if (done == 1) {
            float *snap = s.snap[blockIdx.x];
            for (int i = threadIdx.x; i < a.n_vocab; i += blockDim.x) snap[i] = c.logits[i];
            if (threadIdx.x == 0) { r.snap = *c.state; r.done = 2; }
        }
        if (threadIdx.x == 0 && c.slot) {   // (after the snapshot: tokens[0] is that of the state it saved)
            const int last = r.n_fed - 1;
            c.slot->n_past = c.n_past0 + last;
            c.state->tokens[0] = c.ids[last];
        }
        return false;
    }
    return true;
}
// the id a step of the stopping kernels feeds, and the stop checks on it: the text (or `end`), then the budget
template <class A, class S>
__device__ __forceinline__ void until_feed(const A &a, const S &s, const SampleCtx &c, UntilState &r, int id, bool greedy, bool end = false) {
    feed(a, c, id, greedy);
    r.n_fed = a.step + 1;
    if (reply_take(r, s.tab, id) || end) r.done = 1;
    else if (r.n_fed == r.budget) { r.done = 1; r.by_budget = 1; }
}

// the stop parameter of a stopping kernel: the one element of its parameter pack
template <class S> __device__ __forceinline__ const S &stop_args(const S &s) { return s; }

// ---------------------------------------------------------------------------------------------------------------------------------
// one sampling step of n contexts: grid n, block kThreads.  CTA i samples context i's logits (kMirostat: the mirostat step), writes the
// id into tokens[0] and ids[step], and moves a batched column to its next position.  N is the capacity of the column tables: 8 for up to
// 8 contexts, kMaxBatch above; every column computes the same whatever N.  With a stop parameter (S: StopArgsN<N>) it is sample_until's
// step, which stops each context on its reply's text or its budget.  The stop parameter comes after every parameter of the plain step,
// so those keep their offsets.
// ---------------------------------------------------------------------------------------------------------------------------------
template <int N, bool kMirostat, class... S>
__global__ void __launch_bounds__(kThreads) sample_kernel(const SampleArgsN<N> a, const S... s) {
    const SampleCtx &c = a.c[blockIdx.x];
    const auto step = [&](auto fed) {
        if constexpr (kMirostat) mirostat_body(a, c, mirostat_state(c), fed);
        else sample_body(a, c, fed);
    };
    if constexpr (sizeof...(S) == 0) {
        step([&](int id, bool greedy) { feed(a, c, id, greedy); });
    } else {
        const StopArgsN<N> &st = stop_args(s...);
        UntilState &r = *st.r[blockIdx.x];
        __shared__ int sh_state;
        if (!until_running(a, st, c, r, sh_state)) return;
        step([&](int id, bool greedy) { until_feed(a, st, c, r, id, greedy); });
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// constrained sampling (minigpt4_b200_constraint_*, DESIGN.md §4.12): the twin of sample_kernel's chain that takes each column's
// constraint table.  A constrained column samples over its state's allowed ids only and thread 0 moves its state after feeding; an
// unconstrained column (off null) runs exactly what sample_kernel runs, so one launch takes a mix of both.
// ---------------------------------------------------------------------------------------------------------------------------------
struct ConsCol {
    const int *off;      // the table's row offsets (n_states + 2; row n_states the finished state); null: unconstrained
    const int2 *tr;      // its (id, next state) pairs
    int *state;          // the column's state, which the host uploads before the call
};
template <int N> struct ConsArgsN { ConsCol c[N]; };
static_assert(sizeof(SampleArgsN<LlamaDevice::kMaxBatch>) + sizeof(StopArgsN<LlamaDevice::kMaxBatch>) + sizeof(ConsArgsN<LlamaDevice::kMaxBatch>) <= 32764,
              "the widest constrained kernel's parameters fit the 32 764-byte limit");

// the candidates of column k in its current state (read by every thread before thread 0 can write the next one)
template <class A> __device__ __forceinline__ AllowedIds allowed_ids(const A &a, const ConsCol &k) {
    if (!k.off) return AllowedIds{nullptr, a.n_vocab};
    const int s = *k.state, o = k.off[s];
    return AllowedIds{k.tr + o, k.off[s + 1] - o};
}
template <class A> __device__ __forceinline__ ListedArgs listed_args(const A &a, const AllowedIds &src) { return ListedArgs{a.n_vocab, src}; }
// thread 0, after the draw: the state the fed id leads to (a binary search for it in the row)
__device__ __forceinline__ void cons_advance(const ConsCol &k, const AllowedIds &src, int id) {
    if (!src.listed()) return;
    int lo = 0, hi = src.n - 1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (src.tr[mid].x < id) lo = mid + 1;
        else hi = mid;
    }
    *k.state = src.tr[lo].y;
}

template <class A, class K> __device__ __forceinline__ void sample_cons_step(const A &a, const K &k) {
    const SampleCtx &c = a.c[blockIdx.x];
    const ConsCol &kc = k.c[blockIdx.x];
    const AllowedIds src = allowed_ids(a, kc);
    sample_body(listed_args(a, src), c, [&](int id, bool greedy) { feed(a, c, id, greedy); cons_advance(kc, src, id); });
}
// sample_until's step on a constrained column also stops it after the step that feeds id 2 (</s>)
template <class A, class S, class K> __device__ __forceinline__ void sample_until_cons_step(const A &a, const S &s, const K &k) {
    const SampleCtx &c = a.c[blockIdx.x];
    const ConsCol &kc = k.c[blockIdx.x];
    UntilState &r = *s.r[blockIdx.x];
    __shared__ int sh_state;
    if (!until_running(a, s, c, r, sh_state)) return;
    const AllowedIds src = allowed_ids(a, kc);
    sample_body(listed_args(a, src), c, [&](int id, bool greedy) {
        until_feed(a, s, c, r, id, greedy, src.listed() && id == 2);
        cons_advance(kc, src, id);
    });
}
// the constrained step (S: none) or sample_until's (S: StopArgsN<N>, before the constraint tables as sample_until_cons_step takes them)
template <int N, class... S>
__global__ void __launch_bounds__(kThreads) sample_cons_kernel(const SampleArgsN<N> a, const S... s, const ConsArgsN<N> k) {
    if constexpr (sizeof...(S) == 0) sample_cons_step(a, k);
    else sample_until_cons_step(a, stop_args(s...), k);
}

// seam: reply_take over ids[0, n) from r's tail; *stop_at = the index of the id that ends the reply, -1 if none does
__global__ void reply_check_kernel(ReplyState *r, TokenTable t, const int *ids, int n, int *stop_at) {
    int at = -1;
    for (int i = 0; i < n && at < 0; ++i) if (reply_take(*r, t, ids[i])) at = i;
    *stop_at = at;
}

}  // namespace smp
}  // namespace mg4

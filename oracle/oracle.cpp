// oracle.cpp — CPU restatement of the reference's arithmetic for the hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing in the product (minigpt4_cpp_b200/, libminigpt4.so)
// may include, link or call this file; only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs use it, as the checker / CPU timing arm.
//
// PARITY UNPINNED: the reference (Maknee/minigpt4.cpp @2075cd3) ships no tests, golden
// vectors or fixtures, and its arithmetic lives in a third-party dependency that is not
// on disk: ggerganov/llama.cpp @ tag master-31cfbb1 (bundled ggml.c, k_quants.c, llama.cpp),
// pinned at reference CMakeLists.txt:317-318.  This file restates that revision's published
// algorithms (SURVEY.md §A.3/§B.3) and follows the reference's own graph wiring:
//   * vision graph     : reference minigpt4.cpp:2094-2363 + layer functors :1014-1463
//   * language graph   : llama.cpp llama_eval_internal, called at minigpt4.cpp:2373, :2412
// Block codecs are cross-checked against gguf-py quants.py and the model wiring against
// transformers' Blip2/Llama float models by tests/test_oracle_*.py (not the parity target,
// an independent sanity pin).
//
// FLOAT REDUCTION ORDER.  ggml leaves the order of float accumulation to the build (AVX2 sums in 8 lanes, AVX-512 in 16,
// NEON in 4, scalar in 1, and the thread count changes nothing only because each dot is single-threaded).  Because the
// Q8 activation quantisers are discontinuous, a 1-ulp difference in a matvec output is amplified to ~1e-2 in the logits
// of a deep model (measured, DESIGN.md "Conditioning"), so token-level parity needs ONE fixed order.  For the language
// path this file therefore fixes a canonical "32-lane strided + xor-butterfly" order (lane l accumulates blocks
// l, l+32, ... in increasing order; lanes are combined with offsets 16,8,4,2,1) — i.e. what a 32-wide SIMD build of ggml
// would do — and the CUDA kernels implement exactly the same order, which makes logits bit-identical.  All formulas,
// rounding points, integer block dots and table lookups are ggml's.  FP contraction is disabled on both sides
// (-ffp-contract=off here, -fmad=false in nvcc); FMAs appear only where written explicitly (fmaf), as in ggml's
// _mm256_fmadd_ps sites.  The vision graph keeps the AVX2-shaped order (tensor-core accumulation order is not
// reproducible anyway; it has no quantisers and agrees to ~3e-4).
//
// Build: g++ -O3 -mavx2 -mfma -mf16c -ffp-contract=off -fopenmp -shared -fPIC (the reference's default ISA
// set, reference CMakeLists.txt:27-30,218-227).
#include <immintrin.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <omp.h>
#include <map>
#include <string>
#include <vector>

#define ORACLE_API extern "C" __attribute__((visibility("default")))

typedef uint16_t f16_t;
static inline float h2f(f16_t h) { return _cvtsh_ss(h); }
static inline f16_t f2h(float f) { return _cvtss_sh(f, 0); }  // round-to-nearest-even

// ggml type ids (ggml.h enum ggml_type at master-31cfbb1)
enum { T_F32 = 0, T_F16 = 1, T_Q4_0 = 2, T_Q4_1 = 3, T_Q5_0 = 6, T_Q5_1 = 7, T_Q8_0 = 8, T_Q4_K = 12, T_Q5_K = 13, T_Q6_K = 14 };

#define QK 32
#define QK_K 256

#pragma pack(push, 1)
struct block_q4_0 { f16_t d; uint8_t qs[16]; };                          // 18 B
struct block_q4_1 { f16_t d; f16_t m; uint8_t qs[16]; };                 // 20 B
struct block_q5_0 { f16_t d; uint8_t qh[4]; uint8_t qs[16]; };           // 22 B
struct block_q5_1 { f16_t d; f16_t m; uint8_t qh[4]; uint8_t qs[16]; };  // 24 B
struct block_q8_0 { f16_t d; int8_t qs[32]; };                           // 34 B
struct block_q8_1 { float d; float s; int8_t qs[32]; };                  // 40 B (d,s are F32 at this revision)
struct block_q4_K { f16_t d; f16_t dmin; uint8_t scales[12]; uint8_t qs[128]; };                  // 144 B
struct block_q5_K { f16_t d; f16_t dmin; uint8_t scales[12]; uint8_t qh[32]; uint8_t qs[128]; }; // 176 B
struct block_q6_K { uint8_t ql[128]; uint8_t qh[64]; int8_t scales[16]; f16_t d; };             // 210 B
struct block_q8_K { float d; int8_t qs[256]; int16_t bsums[16]; };        // 292 B
#pragma pack(pop)

// ---------------------------------------------------------------------------------------------
// fp16 lookup tables (ggml.c: table_gelu_f16 / table_silu_f16 / table_exp_f16, built in ggml_init)
// ---------------------------------------------------------------------------------------------
static f16_t g_tab_gelu[65536], g_tab_silu[65536], g_tab_exp[65536];
static bool g_init = false;

static inline float gelu_f32(float x) {
    const float GELU_COEF_A = 0.044715f, SQRT_2_OVER_PI = 0.79788456080286535587989211986876f;
    return 0.5f * x * (1.0f + tanhf(SQRT_2_OVER_PI * x * (1.0f + GELU_COEF_A * x * x)));
}
static inline float silu_f32(float x) { return x / (1.0f + expf(-x)); }

ORACLE_API void oracle_init(void) {
    if (g_init) return;
    for (int i = 0; i < 65536; ++i) {
        float f = h2f((f16_t)i);
        g_tab_gelu[i] = f2h(gelu_f32(f));
        g_tab_silu[i] = f2h(silu_f32(f));
        g_tab_exp[i] = f2h(expf(f));
    }
    g_init = true;
}
// raw table export (tests pin the GPU LUTs against these)
ORACLE_API const uint16_t *oracle_table(int which) {
    oracle_init();
    return which == 0 ? g_tab_gelu : which == 1 ? g_tab_silu : g_tab_exp;
}

// ---------------------------------------------------------------------------------------------
// activation quantisers (ggml.c quantize_row_q8_0 / q8_1 AVX2 semantics; k_quants.c quantize_row_q8_K)
// ---------------------------------------------------------------------------------------------
static inline int rne(float v) { return (int)nearbyintf(v); }  // default rounding mode = nearest-even (== _mm256_round_ps NEAREST)

static void quantize_row_q8_0(const float *x, block_q8_0 *y, int k) {
    for (int i = 0; i < k / QK; ++i) {
        float amax = 0.f;
        for (int j = 0; j < QK; ++j) amax = fmaxf(amax, fabsf(x[i * QK + j]));
        const float d = amax / 127.f;
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        y[i].d = f2h(d);
        for (int j = 0; j < QK; ++j) y[i].qs[j] = (int8_t)rne(x[i * QK + j] * id);
    }
}
static void quantize_row_q8_1(const float *x, block_q8_1 *y, int k) {
    for (int i = 0; i < k / QK; ++i) {
        float amax = 0.f;
        for (int j = 0; j < QK; ++j) amax = fmaxf(amax, fabsf(x[i * QK + j]));
        const float d = amax / 127.f;
        const float id = (amax != 0.0f) ? 127.f / amax : 0.0f;
        y[i].d = d;
        int sum = 0;
        for (int j = 0; j < QK; ++j) { int q = rne(x[i * QK + j] * id); y[i].qs[j] = (int8_t)q; sum += q; }
        y[i].s = d * (float)sum;
    }
}
static inline int nearest_int(float fval) {  // k_quants.c nearest_int: magic-number RNE
    float val = fval + 12582912.f; int i; memcpy(&i, &val, sizeof(int));
    return (i & 0x007fffff) - 0x00400000;
}
static void quantize_row_q8_K(const float *x, block_q8_K *y, int k) {
    for (int i = 0; i < k / QK_K; ++i) {
        float max = 0, amax = 0;
        for (int j = 0; j < QK_K; ++j) { float ax = fabsf(x[j]); if (ax > amax) { amax = ax; max = x[j]; } }
        if (!amax) { y[i].d = 0; memset(y[i].qs, 0, QK_K); memset(y[i].bsums, 0, sizeof(y[i].bsums)); x += QK_K; continue; }
        const float iscale = -128.f / max;
        for (int j = 0; j < QK_K; ++j) { int v = nearest_int(iscale * x[j]); y[i].qs[j] = (int8_t)(v < 127 ? v : 127); }
        for (int j = 0; j < QK_K / 16; ++j) { int s = 0; for (int ii = 0; ii < 16; ++ii) s += y[i].qs[j * 16 + ii]; y[i].bsums[j] = (int16_t)s; }
        y[i].d = 1 / iscale;
        x += QK_K;
    }
}

// ---------------------------------------------------------------------------------------------
// block dot products (ggml.c ggml_vec_dot_q4_0_q8_0 / q4_1_q8_1; k_quants.c ggml_vec_dot_q5_K_q8_K / q6_K_q8_K)
// integer part is exact; float accumulation follows the 8-lane AVX2 shape (acc lanes, then hsum)
// ---------------------------------------------------------------------------------------------
static inline int dot_q4_block(const uint8_t *qs, const int8_t *q8, int bias) {
    int sumi = 0;
    for (int j = 0; j < 16; ++j) {
        sumi += ((qs[j] & 0x0F) - bias) * q8[j] + ((qs[j] >> 4) - bias) * q8[j + 16];
    }
    return sumi;
}
#if defined(__AVX2__)
static inline __m256i bytes_from_nibbles_32(const uint8_t *rsi) {
    const __m128i tmp = _mm_loadu_si128((const __m128i *)rsi);
    const __m256i bytes = _mm256_set_m128i(_mm_srli_epi16(tmp, 4), tmp);
    return _mm256_and_si256(_mm256_set1_epi8(0xF), bytes);
}
static inline __m256 mul_sum_us8_pairs_float(const __m256i ax, const __m256i sy) {
    const __m256i dot = _mm256_maddubs_epi16(ax, sy);
    const __m256i summed = _mm256_madd_epi16(_mm256_set1_epi16(1), dot);
    return _mm256_cvtepi32_ps(summed);
}
static inline float hsum_float_8(const __m256 x) {
    __m128 res = _mm256_extractf128_ps(x, 1);
    res = _mm_add_ps(res, _mm256_castps256_ps128(x));
    res = _mm_add_ps(res, _mm_movehl_ps(res, res));
    res = _mm_add_ss(res, _mm_movehdup_ps(res));
    return _mm_cvtss_f32(res);
}
#endif

static float vec_dot_q4_1_q8_1(int n, const block_q4_1 *x, const block_q8_1 *y) {
    const int nb = n / QK;
#if defined(__AVX2__)
    __m256 acc = _mm256_setzero_ps();
    float summs = 0;
    for (int i = 0; i < nb; ++i) {
        const float d0 = h2f(x[i].d), d1 = y[i].d;
        summs += h2f(x[i].m) * y[i].s;
        const __m256 d0d1 = _mm256_set1_ps(d0 * d1);
        const __m256i bx = bytes_from_nibbles_32(x[i].qs);
        const __m256i by = _mm256_loadu_si256((const __m256i *)y[i].qs);
        acc = _mm256_fmadd_ps(d0d1, mul_sum_us8_pairs_float(bx, by), acc);
    }
    return hsum_float_8(acc) + summs;
#else
    float sumf = 0;
    for (int i = 0; i < nb; ++i) sumf += (h2f(x[i].d) * y[i].d) * dot_q4_block(x[i].qs, y[i].qs, 0) + h2f(x[i].m) * y[i].s;
    return sumf;
#endif
}
static float vec_dot_q4_0_q8_0(int n, const block_q4_0 *x, const block_q8_0 *y) {
    const int nb = n / QK;
    float sumf = 0;
    for (int i = 0; i < nb; ++i) sumf += dot_q4_block(x[i].qs, y[i].qs, 8) * h2f(x[i].d) * h2f(y[i].d);
    return sumf;
}
static inline void get_scale_min_k4(int j, const uint8_t *q, uint8_t *d, uint8_t *m) {
    if (j < 4) { *d = q[j] & 63; *m = q[j + 4] & 63; }
    else { *d = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); *m = (q[j + 4] >> 4) | ((q[j - 0] >> 6) << 4); }
}
static float vec_dot_q5_K_q8_K(int n, const block_q5_K *x, const block_q8_K *y) {
    const int nb = n / QK_K;
    float sums[8] = {0}; float sumf = 0;
    int8_t aux8[QK_K]; int16_t aux16[8]; int32_t aux32[8];
    for (int i = 0; i < nb; ++i) {
        const uint8_t *q4 = x[i].qs, *hm = x[i].qh; const int8_t *q8 = y[i].qs;
        memset(aux32, 0, sizeof(aux32));
        int8_t *a = aux8; uint8_t m = 1;
        for (int j = 0; j < QK_K / 64; ++j) {
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)((q4[l] & 0xF) + ((hm[l] & m) ? 16 : 0));
            a += 32; m <<= 1;
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)((q4[l] >> 4) + ((hm[l] & m) ? 16 : 0));
            a += 32; m <<= 1; q4 += 32;
        }
        uint8_t sc[8], mn[8];
        for (int j = 0; j < 8; ++j) get_scale_min_k4(j, x[i].scales, &sc[j], &mn[j]);
        int sumi = 0;
        for (int j = 0; j < QK_K / 16; ++j) sumi += y[i].bsums[j] * mn[j / 2];
        a = aux8; int is = 0;
        for (int j = 0; j < QK_K / 32; ++j) {
            int32_t scale = sc[is++];
            for (int r = 0; r < 4; ++r) {
                for (int l = 0; l < 8; ++l) aux16[l] = (int16_t)(q8[l] * a[l]);
                for (int l = 0; l < 8; ++l) aux32[l] += scale * aux16[l];
                q8 += 8; a += 8;
            }
        }
        const float d = h2f(x[i].d) * y[i].d;
        for (int l = 0; l < 8; ++l) sums[l] += d * aux32[l];
        const float dmin = h2f(x[i].dmin) * y[i].d;
        sumf -= dmin * sumi;
    }
    for (int l = 0; l < 8; ++l) sumf += sums[l];
    return sumf;
}
// k_quants.c ggml_vec_dot_q4_K_q8_K (scalar shape): Q5_K without the fifth bits
static float vec_dot_q4_K_q8_K(int n, const block_q4_K *x, const block_q8_K *y) {
    const int nb = n / QK_K;
    float sums[8] = {0}; float sumf = 0;
    int8_t aux8[QK_K]; int16_t aux16[8]; int32_t aux32[8];
    for (int i = 0; i < nb; ++i) {
        const uint8_t *q4 = x[i].qs; const int8_t *q8 = y[i].qs;
        memset(aux32, 0, sizeof(aux32));
        int8_t *a = aux8;
        for (int j = 0; j < QK_K / 64; ++j) {
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)(q4[l] & 0xF);
            a += 32;
            for (int l = 0; l < 32; ++l) a[l] = (int8_t)(q4[l] >> 4);
            a += 32; q4 += 32;
        }
        uint8_t sc[8], mn[8];
        for (int j = 0; j < 8; ++j) get_scale_min_k4(j, x[i].scales, &sc[j], &mn[j]);
        int sumi = 0;
        for (int j = 0; j < QK_K / 16; ++j) sumi += y[i].bsums[j] * mn[j / 2];
        a = aux8; int is = 0;
        for (int j = 0; j < QK_K / 32; ++j) {
            int32_t scale = sc[is++];
            for (int r = 0; r < 4; ++r) {
                for (int l = 0; l < 8; ++l) aux16[l] = (int16_t)(q8[l] * a[l]);
                for (int l = 0; l < 8; ++l) aux32[l] += scale * aux16[l];
                q8 += 8; a += 8;
            }
        }
        const float d = h2f(x[i].d) * y[i].d;
        for (int l = 0; l < 8; ++l) sums[l] += d * aux32[l];
        const float dmin = h2f(x[i].dmin) * y[i].d;
        sumf -= dmin * sumi;
    }
    for (int l = 0; l < 8; ++l) sumf += sums[l];
    return sumf;
}
static float vec_dot_q6_K_q8_K(int n, const block_q6_K *x, const block_q8_K *y) {
    const int nb = n / QK_K;
    int8_t aux8[QK_K]; int16_t aux16[8]; int32_t aux32[8]; float sums[8] = {0};
    float sumf = 0;
    for (int i = 0; i < nb; ++i) {
        const uint8_t *q4 = x[i].ql, *qh = x[i].qh; const int8_t *q8 = y[i].qs;
        memset(aux32, 0, sizeof(aux32));
        int8_t *a = aux8;
        for (int j = 0; j < QK_K; j += 128) {
            for (int l = 0; l < 32; ++l) {
                a[l + 0] = (int8_t)((q4[l + 0] & 0xF) | (((qh[l] >> 0) & 3) << 4)) - 32;
                a[l + 32] = (int8_t)((q4[l + 32] & 0xF) | (((qh[l] >> 2) & 3) << 4)) - 32;
                a[l + 64] = (int8_t)((q4[l + 0] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32;
                a[l + 96] = (int8_t)((q4[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32;
            }
            a += 128; q4 += 64; qh += 32;
        }
        a = aux8; int is = 0;
        for (int j = 0; j < QK_K / 16; ++j) {
            int scale = x[i].scales[is++];
            for (int r = 0; r < 2; ++r) {
                for (int l = 0; l < 8; ++l) aux16[l] = (int16_t)(q8[l] * a[l]);
                for (int l = 0; l < 8; ++l) aux32[l] += scale * aux16[l];
                q8 += 8; a += 8;
            }
        }
        const float d = h2f(x[i].d) * y[i].d;
        for (int l = 0; l < 8; ++l) sums[l] += d * aux32[l];
    }
    for (int l = 0; l < 8; ++l) sumf += sums[l];
    return sumf;
}

// F16 dot, F32 accumulate (ggml_vec_dot_f16 with GGML_F16_STEP=32: 4 accumulators x 8 lanes)
static float vec_dot_f16(int n, const f16_t *x, const f16_t *y) {
#if defined(__AVX2__) && defined(__F16C__)
    __m256 s0 = _mm256_setzero_ps(), s1 = s0, s2 = s0, s3 = s0;
    int i = 0;
    const int np = n & ~31;
    for (; i < np; i += 32) {
        s0 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(x + i))), _mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(y + i))), s0);
        s1 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(x + i + 8))), _mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(y + i + 8))), s1);
        s2 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(x + i + 16))), _mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(y + i + 16))), s2);
        s3 = _mm256_fmadd_ps(_mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(x + i + 24))), _mm256_cvtph_ps(_mm_loadu_si128((const __m128i *)(y + i + 24))), s3);
    }
    s0 = _mm256_add_ps(_mm256_add_ps(s0, s1), _mm256_add_ps(s2, s3));
    double sumf = hsum_float_8(s0);
    for (; i < n; ++i) sumf += (double)(h2f(x[i]) * h2f(y[i]));
    return (float)sumf;
#else
    double sumf = 0; for (int i = 0; i < n; ++i) sumf += (double)(h2f(x[i]) * h2f(y[i])); return (float)sumf;
#endif
}
static float vec_dot_f32(int n, const float *x, const float *y) {
#if defined(__AVX2__)
    __m256 s0 = _mm256_setzero_ps(), s1 = s0, s2 = s0, s3 = s0;
    int i = 0; const int np = n & ~31;
    for (; i < np; i += 32) {
        s0 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i), _mm256_loadu_ps(y + i), s0);
        s1 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i + 8), _mm256_loadu_ps(y + i + 8), s1);
        s2 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i + 16), _mm256_loadu_ps(y + i + 16), s2);
        s3 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i + 24), _mm256_loadu_ps(y + i + 24), s3);
    }
    s0 = _mm256_add_ps(_mm256_add_ps(s0, s1), _mm256_add_ps(s2, s3));
    double sumf = hsum_float_8(s0);
    for (; i < n; ++i) sumf += (double)(x[i] * y[i]);
    return (float)sumf;
#else
    double sumf = 0; for (int i = 0; i < n; ++i) sumf += (double)(x[i] * y[i]); return (float)sumf;
#endif
}

// Q5_0 / Q5_1 / Q8_0 (ggml.c ggml_vec_dot_q5_0_q8_0 / q5_1_q8_1 / q8_0_q8_0): the fifth bit of weight j sits in bit j of qh (low half of the
// block) and bit j+16 (high half).  Scalar statement of the block sums; the float accumulation is one running sum per row, as in ggml's
// scalar path (these types are only reached through quantised MiniGPT-4 containers / llama files, never on the bit-exact decode path).
static inline int dot_q5_block(const uint8_t *qs, const uint8_t *qh4, const int8_t *q8, int bias) {
    uint32_t qh; memcpy(&qh, qh4, 4);
    int sumi = 0;
    for (int j = 0; j < 16; ++j) {
        const int x0 = ((qs[j] & 0x0F) | (int)(((qh >> j) & 1u) << 4)) - bias;
        const int x1 = ((qs[j] >> 4) | (int)(((qh >> (j + 16)) & 1u) << 4)) - bias;
        sumi += x0 * q8[j] + x1 * q8[j + 16];
    }
    return sumi;
}
static float vec_dot_q5_0_q8_0(int n, const block_q5_0 *x, const block_q8_0 *y) {
    float sumf = 0;
    for (int i = 0; i < n / QK; ++i) sumf += (h2f(x[i].d) * h2f(y[i].d)) * dot_q5_block(x[i].qs, x[i].qh, y[i].qs, 16);
    return sumf;
}
static float vec_dot_q5_1_q8_1(int n, const block_q5_1 *x, const block_q8_1 *y) {
    float sumf = 0;
    for (int i = 0; i < n / QK; ++i) sumf += (h2f(x[i].d) * y[i].d) * dot_q5_block(x[i].qs, x[i].qh, y[i].qs, 0) + h2f(x[i].m) * y[i].s;
    return sumf;
}
static float vec_dot_q8_0_q8_0(int n, const block_q8_0 *x, const block_q8_0 *y) {
    float sumf = 0;
    for (int i = 0; i < n / QK; ++i) { int sumi = 0; for (int j = 0; j < 32; ++j) sumi += x[i].qs[j] * y[i].qs[j]; sumf += (h2f(x[i].d) * h2f(y[i].d)) * sumi; }
    return sumf;
}
// ---------------------------------------------------------------------------------------------
// canonical-order reductions (language path) — mirrored 1:1 by csrc/llama_kernels.cuh
// ---------------------------------------------------------------------------------------------
template <typename T> static inline T butterfly(T *v, int n) {  // v'[l] = v[l] + v[l ^ o], o = n/2 .. 1 ; returns lane 0
    T t[32];
    for (int o = n / 2; o > 0; o >>= 1) { for (int l = 0; l < n; ++l) t[l] = v[l] + v[l ^ o]; for (int l = 0; l < n; ++l) v[l] = t[l]; }
    return v[0];
}
// block_sum of llama_kernels.cuh: NW warps of 32 partials; warp butterflies, then a butterfly over the NW warp sums
static double block_sum_n(const double *partial, int nw) {
    double w[32];
    for (int l = 0; l < 32; ++l) w[l] = 0.0;
    for (int wi = 0; wi < nw; ++wi) { double v[32]; for (int l = 0; l < 32; ++l) v[l] = partial[wi * 32 + l]; w[wi] = butterfly(v, 32); }
    return butterfly(w, 32);
}
static double block_sum_256(const double *partial /*[256]*/) { return block_sum_n(partial, 8); }

static float dot_canon_q4_1(int n, const block_q4_1 *x, const block_q8_1 *y) {
    const int nb = n / QK;
    float accd[32], accm[32];
#if defined(__AVX2__)
    __m256 A[4], M[4];
    for (int k = 0; k < 4; ++k) { A[k] = _mm256_setzero_ps(); M[k] = _mm256_setzero_ps(); }
    const __m256i ones = _mm256_set1_epi16(1);
    int b0 = 0;
    for (; b0 + 32 <= nb; b0 += 32) {
        for (int k = 0; k < 4; ++k) {
            __m256i s[8]; float dd[8] __attribute__((aligned(32))), mm[8] __attribute__((aligned(32))), ss[8] __attribute__((aligned(32)));
            for (int j = 0; j < 8; ++j) {
                const int b = b0 + 8 * k + j;
                const __m256i bx = bytes_from_nibbles_32(x[b].qs), by = _mm256_loadu_si256((const __m256i *)y[b].qs);
                s[j] = _mm256_madd_epi16(ones, _mm256_maddubs_epi16(bx, by));
                dd[j] = h2f(x[b].d) * y[b].d; mm[j] = h2f(x[b].m); ss[j] = y[b].s;
            }
            const __m256i t0 = _mm256_hadd_epi32(s[0], s[1]), t1 = _mm256_hadd_epi32(s[2], s[3]), t2 = _mm256_hadd_epi32(s[4], s[5]), t3 = _mm256_hadd_epi32(s[6], s[7]);
            const __m256i u0 = _mm256_hadd_epi32(t0, t1), u1 = _mm256_hadd_epi32(t2, t3);
            const __m256i tot = _mm256_add_epi32(_mm256_permute2x128_si256(u0, u1, 0x20), _mm256_permute2x128_si256(u0, u1, 0x31));
            A[k] = _mm256_fmadd_ps(_mm256_load_ps(dd), _mm256_cvtepi32_ps(tot), A[k]);
            M[k] = _mm256_fmadd_ps(_mm256_load_ps(mm), _mm256_load_ps(ss), M[k]);
        }
    }
    for (int k = 0; k < 4; ++k) { _mm256_storeu_ps(accd + 8 * k, A[k]); _mm256_storeu_ps(accm + 8 * k, M[k]); }
    for (int b = b0; b < nb; ++b) {  // ragged tail: lane = b mod 32
        const int l = b & 31;
        accd[l] = fmaf(h2f(x[b].d) * y[b].d, (float)dot_q4_block(x[b].qs, y[b].qs, 0), accd[l]);
        accm[l] = fmaf(h2f(x[b].m), y[b].s, accm[l]);
    }
#else
    for (int l = 0; l < 32; ++l) { accd[l] = 0.f; accm[l] = 0.f; }
    for (int b = 0; b < nb; ++b) { const int l = b & 31;
        accd[l] = fmaf(h2f(x[b].d) * y[b].d, (float)dot_q4_block(x[b].qs, y[b].qs, 0), accd[l]); accm[l] = fmaf(h2f(x[b].m), y[b].s, accm[l]); }
#endif
    const float sd = butterfly(accd, 32), sm = butterfly(accm, 32);
    return sd + sm;
}
static float dot_canon_q4_0(int n, const block_q4_0 *x, const block_q8_0 *y) {
    const int nb = n / QK;
    float acc[32];
    for (int l = 0; l < 32; ++l) acc[l] = 0.f;
    for (int b = 0; b < nb; ++b) { const int l = b & 31; acc[l] += ((float)dot_q4_block(x[b].qs, y[b].qs, 8) * h2f(x[b].d)) * h2f(y[b].d); }
    return butterfly(acc, 32);
}
// K-quants: 8 lanes per super-block, 4 super-blocks per warp pass (lane = 8*(sb%4) + part)
static float dot_canon_q5_K(int n, const block_q5_K *x, const block_q8_K *y) {
    const int nsb = n / QK_K;
    float accd[32], accm[32];
    for (int l = 0; l < 32; ++l) { accd[l] = 0.f; accm[l] = 0.f; }
    for (int sb = 0; sb < nsb; ++sb) {
        const float d = h2f(x[sb].d), dmin = h2f(x[sb].dmin), d8 = y[sb].d;
        for (int part = 0; part < 8; ++part) {
            const int l = 8 * (sb & 3) + part, j = part >> 1, hf = part & 1;
            uint8_t sca, mna, scb, mnb;
            get_scale_min_k4(2 * j, x[sb].scales, &sca, &mna); get_scale_min_k4(2 * j + 1, x[sb].scales, &scb, &mnb);
            int s0 = 0, s1 = 0;
            for (int i = 0; i < 16; ++i) {
                const uint8_t qb = x[sb].qs[32 * j + 16 * hf + i], hb = x[sb].qh[16 * hf + i];
                const int lo = (qb & 0xF) + (((hb >> (2 * j)) & 1) << 4), hi = (qb >> 4) + (((hb >> (2 * j + 1)) & 1) << 4);
                s0 += lo * y[sb].qs[64 * j + 16 * hf + i]; s1 += hi * y[sb].qs[64 * j + 32 + 16 * hf + i];
            }
            accd[l] += (d * d8) * (float)(sca * s0 + scb * s1);
            accm[l] += (dmin * d8) * (float)(mna * y[sb].bsums[4 * j + hf] + mnb * y[sb].bsums[4 * j + 2 + hf]);
        }
    }
    const float sd = butterfly(accd, 32), sm = butterfly(accm, 32);
    return sd - sm;
}
// Q4_K: the Q5_K canonical order without the fifth bits (8 lanes per super-block, 4 super-blocks per warp pass)
static float dot_canon_q4_K(int n, const block_q4_K *x, const block_q8_K *y) {
    const int nsb = n / QK_K;
    float accd[32], accm[32];
    for (int l = 0; l < 32; ++l) { accd[l] = 0.f; accm[l] = 0.f; }
    for (int sb = 0; sb < nsb; ++sb) {
        const float d = h2f(x[sb].d), dmin = h2f(x[sb].dmin), d8 = y[sb].d;
        for (int part = 0; part < 8; ++part) {
            const int l = 8 * (sb & 3) + part, j = part >> 1, hf = part & 1;
            uint8_t sca, mna, scb, mnb;
            get_scale_min_k4(2 * j, x[sb].scales, &sca, &mna); get_scale_min_k4(2 * j + 1, x[sb].scales, &scb, &mnb);
            int s0 = 0, s1 = 0;
            for (int i = 0; i < 16; ++i) {
                const uint8_t qb = x[sb].qs[32 * j + 16 * hf + i];
                s0 += (qb & 0xF) * y[sb].qs[64 * j + 16 * hf + i]; s1 += (qb >> 4) * y[sb].qs[64 * j + 32 + 16 * hf + i];
            }
            accd[l] += (d * d8) * (float)(sca * s0 + scb * s1);
            accm[l] += (dmin * d8) * (float)(mna * y[sb].bsums[4 * j + hf] + mnb * y[sb].bsums[4 * j + 2 + hf]);
        }
    }
    const float sd = butterfly(accd, 32), sm = butterfly(accm, 32);
    return sd - sm;
}
// Q5_0 / Q5_1 / Q8_0 in the canonical 32-lane strided order (the shapes of dot_canon_q4_0 / q4_1): the specification the CUDA kernels
// for these types will have to meet bit for bit
static float dot_canon_q5_0(int n, const block_q5_0 *x, const block_q8_0 *y) {
    float acc[32];
    for (int l = 0; l < 32; ++l) acc[l] = 0.f;
    for (int b = 0; b < n / QK; ++b) { const int l = b & 31; acc[l] += ((float)dot_q5_block(x[b].qs, x[b].qh, y[b].qs, 16) * h2f(x[b].d)) * h2f(y[b].d); }
    return butterfly(acc, 32);
}
static float dot_canon_q5_1(int n, const block_q5_1 *x, const block_q8_1 *y) {
    float accd[32], accm[32];
    for (int l = 0; l < 32; ++l) { accd[l] = 0.f; accm[l] = 0.f; }
    for (int b = 0; b < n / QK; ++b) { const int l = b & 31;
        accd[l] = fmaf(h2f(x[b].d) * y[b].d, (float)dot_q5_block(x[b].qs, x[b].qh, y[b].qs, 0), accd[l]); accm[l] = fmaf(h2f(x[b].m), y[b].s, accm[l]); }
    const float sd = butterfly(accd, 32), sm = butterfly(accm, 32);
    return sd + sm;
}
static float dot_canon_q8_0(int n, const block_q8_0 *x, const block_q8_0 *y) {
    float acc[32];
    for (int l = 0; l < 32; ++l) acc[l] = 0.f;
    for (int b = 0; b < n / QK; ++b) { const int l = b & 31; int sumi = 0; for (int j = 0; j < 32; ++j) sumi += x[b].qs[j] * y[b].qs[j];
        acc[l] += ((float)sumi * h2f(x[b].d)) * h2f(y[b].d); }
    return butterfly(acc, 32);
}
static float dot_canon_q6_K(int n, const block_q6_K *x, const block_q8_K *y) {
    const int nsb = n / QK_K;
    float acc[32];
    for (int l = 0; l < 32; ++l) acc[l] = 0.f;
    for (int sb = 0; sb < nsb; ++sb) {
        const float d = h2f(x[sb].d), d8 = y[sb].d;
        for (int part = 0; part < 8; ++part) {
            const int l = 8 * (sb & 3) + part, nn = part >> 2, u = part & 3;
            int isum = 0;
            for (int kq = 0; kq < 4; ++kq) {
                int s = 0;
                for (int i = 0; i < 8; ++i) {
                    const int li = 8 * u + i;
                    const uint8_t lb = x[sb].ql[64 * nn + (kq & 1) * 32 + li];
                    const int nib = (kq >= 2) ? (lb >> 4) : (lb & 0xF);
                    const int hb = (x[sb].qh[32 * nn + li] >> (2 * kq)) & 3;
                    s += ((nib | (hb << 4)) - 32) * y[sb].qs[128 * nn + 32 * kq + li];
                }
                isum += x[sb].scales[8 * nn + 2 * kq + (u >> 1)] * s;
            }
            acc[l] += (d * d8) * (float)isum;
        }
    }
    return butterfly(acc, 32);
}
// F16 weights: lane l owns 8-element vectors l, l+32, ... ; inside a vector elements are accumulated in order with FMA
static float dot_canon_f16(int n, const f16_t *x, const f16_t *y) {
    const int nv = n / 8;
    float acc[32];
    for (int l = 0; l < 32; ++l) acc[l] = 0.f;
    for (int v = 0; v < nv; ++v) { const int l = v & 31; for (int e = 0; e < 8; ++e) acc[l] = fmaf(h2f(x[8 * v + e]), h2f(y[8 * v + e]), acc[l]); }
    return butterfly(acc, 32);
}

// ---------------------------------------------------------------------------------------------
// generic tensor + mul_mat (ggml_compute_forward_mul_mat dispatch, SURVEY §A.3)
// W: [rows][cols] in `type`; X: F32 [n][cols]; Y: F32 [n][rows].  Y[n][r] = dot(W[r], X[n])
// ---------------------------------------------------------------------------------------------
struct Tensor { int type; int64_t ne[4]; const void *data; };

static size_t row_bytes(int type, int64_t cols) {
    switch (type) {
        case T_F32: return cols * 4; case T_F16: return cols * 2;
        case T_Q4_0: return cols / 32 * 18; case T_Q4_1: return cols / 32 * 20;
        case T_Q5_0: return cols / 32 * 22; case T_Q5_1: return cols / 32 * 24; case T_Q8_0: return cols / 32 * 34;
        case T_Q4_K: return cols / 256 * 144; case T_Q5_K: return cols / 256 * 176; case T_Q6_K: return cols / 256 * 210;
    }
    fprintf(stderr, "oracle: unsupported type %d\n", type); abort();
}

static void mul_mat(const Tensor &W, const float *X, int n, float *Y, bool canon = false) {
    const int64_t cols = W.ne[0], rows = W.ne[1];
    const size_t rb = row_bytes(W.type, cols);
    const uint8_t *wd = (const uint8_t *)W.data;
    if (W.type == T_F32) {
#pragma omp parallel for schedule(static)
        for (int64_t r = 0; r < rows; ++r)
            for (int i = 0; i < n; ++i) Y[(size_t)i * rows + r] = vec_dot_f32((int)cols, (const float *)(wd + r * rb), X + (size_t)i * cols);
        return;
    }
    // quantise / convert the activation rows to the weight type's vec_dot_type
    size_t qrb;
    switch (W.type) {
        case T_F16: qrb = cols * 2; break;
        case T_Q4_0: case T_Q5_0: case T_Q8_0: qrb = cols / 32 * sizeof(block_q8_0); break;
        case T_Q4_1: case T_Q5_1: qrb = cols / 32 * sizeof(block_q8_1); break;
        default: qrb = cols / 256 * sizeof(block_q8_K); break;
    }
    std::vector<uint8_t> wdata(qrb * (size_t)n);
#pragma omp parallel for schedule(static)
    for (int i = 0; i < n; ++i) {
        const float *x = X + (size_t)i * cols; uint8_t *q = wdata.data() + qrb * i;
        switch (W.type) {
            case T_F16: for (int64_t c = 0; c < cols; ++c) ((f16_t *)q)[c] = f2h(x[c]); break;
            case T_Q4_0: case T_Q5_0: case T_Q8_0: quantize_row_q8_0(x, (block_q8_0 *)q, (int)cols); break;
            case T_Q4_1: case T_Q5_1: quantize_row_q8_1(x, (block_q8_1 *)q, (int)cols); break;
            default: quantize_row_q8_K(x, (block_q8_K *)q, (int)cols); break;
        }
    }
#pragma omp parallel for schedule(static)
    for (int64_t r = 0; r < rows; ++r) {
        const uint8_t *w = wd + r * rb;
        for (int i = 0; i < n; ++i) {
            const uint8_t *q = wdata.data() + qrb * i; float v;
            if (W.type == T_Q5_0) v = canon ? dot_canon_q5_0((int)cols, (const block_q5_0 *)w, (const block_q8_0 *)q) : vec_dot_q5_0_q8_0((int)cols, (const block_q5_0 *)w, (const block_q8_0 *)q);
            else if (W.type == T_Q5_1) v = canon ? dot_canon_q5_1((int)cols, (const block_q5_1 *)w, (const block_q8_1 *)q) : vec_dot_q5_1_q8_1((int)cols, (const block_q5_1 *)w, (const block_q8_1 *)q);
            else if (W.type == T_Q8_0) v = canon ? dot_canon_q8_0((int)cols, (const block_q8_0 *)w, (const block_q8_0 *)q) : vec_dot_q8_0_q8_0((int)cols, (const block_q8_0 *)w, (const block_q8_0 *)q);
            else if (W.type == T_Q4_K) v = canon ? dot_canon_q4_K((int)cols, (const block_q4_K *)w, (const block_q8_K *)q) : vec_dot_q4_K_q8_K((int)cols, (const block_q4_K *)w, (const block_q8_K *)q);
            else if (canon) switch (W.type) {
                case T_F16: v = dot_canon_f16((int)cols, (const f16_t *)w, (const f16_t *)q); break;
                case T_Q4_0: v = dot_canon_q4_0((int)cols, (const block_q4_0 *)w, (const block_q8_0 *)q); break;
                case T_Q4_1: v = dot_canon_q4_1((int)cols, (const block_q4_1 *)w, (const block_q8_1 *)q); break;
                case T_Q5_K: v = dot_canon_q5_K((int)cols, (const block_q5_K *)w, (const block_q8_K *)q); break;
                default: v = dot_canon_q6_K((int)cols, (const block_q6_K *)w, (const block_q8_K *)q); break;
            } else switch (W.type) {
                case T_F16: v = vec_dot_f16((int)cols, (const f16_t *)w, (const f16_t *)q); break;
                case T_Q4_0: v = vec_dot_q4_0_q8_0((int)cols, (const block_q4_0 *)w, (const block_q8_0 *)q); break;
                case T_Q4_1: v = vec_dot_q4_1_q8_1((int)cols, (const block_q4_1 *)w, (const block_q8_1 *)q); break;
                case T_Q5_K: v = vec_dot_q5_K_q8_K((int)cols, (const block_q5_K *)w, (const block_q8_K *)q); break;
                default: v = vec_dot_q6_K_q8_K((int)cols, (const block_q6_K *)w, (const block_q8_K *)q); break;
            }
            Y[(size_t)i * rows + r] = v;
        }
    }
}

// dequantise one row to F32 (ggml_get_rows on a quantised matrix; dequantize_row_*)
static void dequant_row(const Tensor &W, int64_t r, float *y) {
    const int64_t cols = W.ne[0];
    const uint8_t *w = (const uint8_t *)W.data + r * row_bytes(W.type, cols);
    switch (W.type) {
        case T_F32: memcpy(y, w, cols * 4); break;
        case T_F16: for (int64_t c = 0; c < cols; ++c) y[c] = h2f(((const f16_t *)w)[c]); break;
        case T_Q4_0: { const block_q4_0 *b = (const block_q4_0 *)w;
            for (int i = 0; i < cols / 32; ++i) { float d = h2f(b[i].d);
                for (int j = 0; j < 16; ++j) { y[i * 32 + j] = ((b[i].qs[j] & 0xF) - 8) * d; y[i * 32 + j + 16] = ((b[i].qs[j] >> 4) - 8) * d; } } } break;
        case T_Q4_1: { const block_q4_1 *b = (const block_q4_1 *)w;
            for (int i = 0; i < cols / 32; ++i) { float d = h2f(b[i].d), m = h2f(b[i].m);
                for (int j = 0; j < 16; ++j) { y[i * 32 + j] = (b[i].qs[j] & 0xF) * d + m; y[i * 32 + j + 16] = (b[i].qs[j] >> 4) * d + m; } } } break;
        case T_Q5_0: { const block_q5_0 *b = (const block_q5_0 *)w;
            for (int i = 0; i < cols / 32; ++i) { const float d = h2f(b[i].d); uint32_t qh; memcpy(&qh, b[i].qh, 4);
                for (int j = 0; j < 16; ++j) {
                    y[i * 32 + j] = (((b[i].qs[j] & 0xF) | (int)(((qh >> j) & 1u) << 4)) - 16) * d;
                    y[i * 32 + j + 16] = (((b[i].qs[j] >> 4) | (int)(((qh >> (j + 16)) & 1u) << 4)) - 16) * d; } } } break;
        case T_Q5_1: { const block_q5_1 *b = (const block_q5_1 *)w;
            for (int i = 0; i < cols / 32; ++i) { const float d = h2f(b[i].d), m = h2f(b[i].m); uint32_t qh; memcpy(&qh, b[i].qh, 4);
                for (int j = 0; j < 16; ++j) {
                    y[i * 32 + j] = ((b[i].qs[j] & 0xF) | (int)(((qh >> j) & 1u) << 4)) * d + m;
                    y[i * 32 + j + 16] = ((b[i].qs[j] >> 4) | (int)(((qh >> (j + 16)) & 1u) << 4)) * d + m; } } } break;
        case T_Q8_0: { const block_q8_0 *b = (const block_q8_0 *)w;
            for (int i = 0; i < cols / 32; ++i) { const float d = h2f(b[i].d); for (int j = 0; j < 32; ++j) y[i * 32 + j] = b[i].qs[j] * d; } } break;
        case T_Q4_K: { const block_q4_K *b = (const block_q4_K *)w;
            for (int i = 0; i < cols / 256; ++i) {
                const uint8_t *ql = b[i].qs; const float d = h2f(b[i].d), min = h2f(b[i].dmin);
                int is = 0; uint8_t sc, m; float *yy = y + i * 256;
                for (int j = 0; j < 256; j += 64) {
                    get_scale_min_k4(is + 0, b[i].scales, &sc, &m); const float d1 = d * sc, m1 = min * m;
                    get_scale_min_k4(is + 1, b[i].scales, &sc, &m); const float d2 = d * sc, m2 = min * m;
                    for (int l = 0; l < 32; ++l) *yy++ = d1 * (ql[l] & 0xF) - m1;
                    for (int l = 0; l < 32; ++l) *yy++ = d2 * (ql[l] >> 4) - m2;
                    ql += 32; is += 2;
                } } } break;
        case T_Q5_K: { const block_q5_K *b = (const block_q5_K *)w;
            for (int i = 0; i < cols / 256; ++i) {
                const uint8_t *ql = b[i].qs, *qh = b[i].qh; const float d = h2f(b[i].d), min = h2f(b[i].dmin);
                int is = 0; uint8_t sc, m; uint8_t u1 = 1, u2 = 2; float *yy = y + i * 256;
                for (int j = 0; j < 256; j += 64) {
                    get_scale_min_k4(is + 0, b[i].scales, &sc, &m); const float d1 = d * sc, m1 = min * m;
                    get_scale_min_k4(is + 1, b[i].scales, &sc, &m); const float d2 = d * sc, m2 = min * m;
                    for (int l = 0; l < 32; ++l) *yy++ = d1 * ((ql[l] & 0xF) + (qh[l] & u1 ? 16 : 0)) - m1;
                    for (int l = 0; l < 32; ++l) *yy++ = d2 * ((ql[l] >> 4) + (qh[l] & u2 ? 16 : 0)) - m2;
                    ql += 32; is += 2; u1 <<= 2; u2 <<= 2;
                } } } break;
        case T_Q6_K: { const block_q6_K *b = (const block_q6_K *)w;
            for (int i = 0; i < cols / 256; ++i) {
                const float d = h2f(b[i].d); const uint8_t *ql = b[i].ql, *qh = b[i].qh; const int8_t *sc = b[i].scales; float *yy = y + i * 256;
                for (int n = 0; n < 256; n += 128) {
                    for (int l = 0; l < 32; ++l) { int is = l / 16;
                        const int8_t q1 = (int8_t)((ql[l + 0] & 0xF) | (((qh[l] >> 0) & 3) << 4)) - 32;
                        const int8_t q2 = (int8_t)((ql[l + 32] & 0xF) | (((qh[l] >> 2) & 3) << 4)) - 32;
                        const int8_t q3 = (int8_t)((ql[l + 0] >> 4) | (((qh[l] >> 4) & 3) << 4)) - 32;
                        const int8_t q4 = (int8_t)((ql[l + 32] >> 4) | (((qh[l] >> 6) & 3) << 4)) - 32;
                        yy[l + 0] = d * sc[is + 0] * q1; yy[l + 32] = d * sc[is + 2] * q2; yy[l + 64] = d * sc[is + 4] * q3; yy[l + 96] = d * sc[is + 6] * q4; }
                    yy += 128; ql += 64; qh += 32; sc += 8;
                } } } break;
        default: abort();
    }
}

// ---------------------------------------------------------------------------------------------
// elementwise / row ops (ggml.c forward kernels at this revision)
// ---------------------------------------------------------------------------------------------
static void op_norm(const float *x, float *y, int n, int rows) {  // ggml_norm, eps 1e-5
#pragma omp parallel for schedule(static)
    for (int r = 0; r < rows; ++r) {
        const float *xr = x + (size_t)r * n; float *yr = y + (size_t)r * n;
        double sum = 0; for (int i = 0; i < n; ++i) sum += (double)xr[i];
        float mean = (float)(sum / n);
        double sum2 = 0; for (int i = 0; i < n; ++i) { float v = xr[i] - mean; yr[i] = v; sum2 += (double)(v * v); }
        float variance = (float)(sum2 / n);
        const float scale = 1.0f / sqrtf(variance + 1e-5f);
        for (int i = 0; i < n; ++i) yr[i] *= scale;
    }
}
static void op_layernorm(const float *x, float *y, int n, int rows, const float *w, const float *b) {  // NNLayerNorm::forward minigpt4.cpp:1074-1093
    op_norm(x, y, n, rows);
    for (int r = 0; r < rows; ++r) for (int i = 0; i < n; ++i) { float v = w[i] * y[(size_t)r * n + i]; y[(size_t)r * n + i] = b ? v + b[i] : v; }
}
static void op_rms_norm_mul(const float *x, float *y, int n, int rows, const float *w) {  // ggml_rms_norm eps 1e-6, then ggml_mul
    for (int r = 0; r < rows; ++r) {
        const float *xr = x + (size_t)r * n; float *yr = y + (size_t)r * n;
        double part[512];  // canonical order: 512 partials; partial p owns elements 2048k + 4p + e (k outer, e = 0..3 inner)
        for (int t = 0; t < 512; ++t) { double s = 0; for (int k = 0; 2048 * k + 4 * t < n; ++k) for (int e = 0; e < 4; ++e) { const int i = 2048 * k + 4 * t + e; if (i < n) s += (double)(xr[i] * xr[i]); } part[t] = s; }
        const double sum = block_sum_n(part, 16);
        const float mean = (float)(sum / n);
        const float scale = 1.0f / sqrtf(mean + 1e-6f);
        for (int i = 0; i < n; ++i) yr[i] = (xr[i] * scale) * w[i];
    }
}
static void op_softmax_row(float *p, int n) {  // ggml_compute_forward_soft_max_f32 (fp16 exp LUT, double sum)
    float max = -INFINITY; for (int i = 0; i < n; ++i) max = fmaxf(max, p[i]);
    double sum = 0;
    for (int i = 0; i < n; ++i) {
        if (p[i] == -INFINITY) { p[i] = 0.0f; }
        else { float val = h2f(g_tab_exp[f2h(p[i] - max)]); sum += (double)val; p[i] = val; }
    }
    const float inv = (float)(1.0 / sum);
    for (int i = 0; i < n; ++i) p[i] *= inv;
}
static inline float op_gelu(float x) { return h2f(g_tab_gelu[f2h(x)]); }
static inline float op_silu(float x) { return h2f(g_tab_silu[f2h(x)]); }

// exported single ops for kernel-level parity tests ------------------------------------------------
ORACLE_API void oracle_mul_mat(int type, int64_t rows, int64_t cols, const void *w, const float *x, int n, float *y) {
    oracle_init(); Tensor W{type, {cols, rows, 1, 1}, w}; mul_mat(W, x, n, y, true);
}
ORACLE_API void oracle_dequant_row(int type, int64_t cols, const void *wrow, float *y) {
    Tensor W{type, {cols, 1, 1, 1}, wrow}; dequant_row(W, 0, y);
}
ORACLE_API void oracle_quantize_q8_1(const float *x, void *y, int k) { quantize_row_q8_1(x, (block_q8_1 *)y, k); }
ORACLE_API void oracle_quantize_q8_0(const float *x, void *y, int k) { quantize_row_q8_0(x, (block_q8_0 *)y, k); }
ORACLE_API void oracle_quantize_q8_K(const float *x, void *y, int k) { quantize_row_q8_K(x, (block_q8_K *)y, k); }
ORACLE_API void oracle_layernorm(const float *x, float *y, int n, int rows, const float *w, const float *b) { op_layernorm(x, y, n, rows, w, b); }
ORACLE_API void oracle_rms_norm_mul(const float *x, float *y, int n, int rows, const float *w) { op_rms_norm_mul(x, y, n, rows, w); }
ORACLE_API void oracle_softmax(float *p, int n, int rows) { oracle_init(); for (int r = 0; r < rows; ++r) op_softmax_row(p + (size_t)r * n, n); }
ORACLE_API void oracle_gelu(const float *x, float *y, int n) { oracle_init(); for (int i = 0; i < n; ++i) y[i] = op_gelu(x[i]); }
ORACLE_API void oracle_silu(const float *x, float *y, int n) { oracle_init(); for (int i = 0; i < n; ++i) y[i] = op_silu(x[i]); }

// ---------------------------------------------------------------------------------------------
// model container handed over from Python (name -> tensor view)
// ---------------------------------------------------------------------------------------------
struct Model { std::map<std::string, Tensor> t; };

ORACLE_API void *oracle_model_new(void) { oracle_init(); return new Model(); }
ORACLE_API void oracle_model_free(void *m) { delete (Model *)m; }
ORACLE_API void oracle_model_add(void *m, const char *name, int type, int ndim, const int64_t *ne, const void *data) {
    Tensor t{type, {1, 1, 1, 1}, data}; for (int i = 0; i < ndim; ++i) t.ne[i] = ne[i];
    ((Model *)m)->t[name] = t;
}
static const Tensor &T(const Model *m, const std::string &name) {
    auto it = m->t.find(name);
    if (it == m->t.end()) { fprintf(stderr, "oracle: missing tensor %s\n", name.c_str()); abort(); }
    return it->second;
}
static const Tensor *Topt(const Model *m, const std::string &name) { auto it = m->t.find(name); return it == m->t.end() ? nullptr : &it->second; }
static const float *F(const Model *m, const std::string &name) { const Tensor &t = T(m, name); if (t.type != T_F32) { fprintf(stderr, "oracle: %s not f32\n", name.c_str()); abort(); } return (const float *)t.data; }

// NNLinear::forward (minigpt4.cpp:1014-1032): mul_mat then bias + result
static void linear(const Model *m, const std::string &prefix, const float *x, int n, float *y) {
    const Tensor &W = T(m, prefix + ".weight");
    mul_mat(W, x, n, y);
    if (const Tensor *b = Topt(m, prefix + ".bias")) {
        const float *bd = (const float *)b->data; const int64_t rows = W.ne[1];
        for (int i = 0; i < n; ++i) for (int64_t r = 0; r < rows; ++r) y[(size_t)i * rows + r] = bd[r] + y[(size_t)i * rows + r];
    }
}

// ---------------------------------------------------------------------------------------------
// vision graph: MiniGPT4::encode_image (minigpt4.cpp:2094-2363)
// image: F32 CHW [3][224][224]; out: F32 [32][n_embd_llm]
// `tap`, when non-NULL, receives intermediate activations for layer-level parity tests:
//   tap_kind 1 = embeddings after pos_embed [T][D]; 2 = after ViT block `tap_idx` [T][D];
//   3 = ln_vision output [T][D]; 4 = Q-Former layer `tap_idx` output [32][768]
// oracle_vit_encode_stages: one run that fills every stage at once (each pointer may be NULL): embed [T][D], vit_blocks [n_blocks][T][D],
//   ln_vision [T][D], qformer [q_layers][32][768], and out
// ---------------------------------------------------------------------------------------------
struct VitStages { float *embed, *vit_blocks, *ln_vision, *qformer; };
struct VitDims { int D, T, H, dh, nblocks, P, patch; };

// NNQKVAttention::forward (minigpt4.cpp:1246-1315)
static void vit_attention(const Model *m, const std::string &pfx, const VitDims &v, const float *x, float *out) {
    const int D = v.D, Tn = v.T, H = v.H, dh = v.dh;
    std::vector<float> qkv((size_t)Tn * 3 * D);
    mul_mat(T(m, pfx + "qkv.weight"), x, Tn, qkv.data());
    const float *qb = F(m, pfx + "q_bias"), *vb = F(m, pfx + "v_bias");
    for (int t = 0; t < Tn; ++t) { float *r = qkv.data() + (size_t)t * 3 * D;
        for (int i = 0; i < D; ++i) { r[i] = qb[i] + r[i]; r[D + i] = 0.0f + r[D + i]; r[2 * D + i] = vb[i] + r[2 * D + i]; } }
    const float scale = 1.0f / sqrtf((float)dh);
    std::vector<float> ctx((size_t)Tn * D);
#pragma omp parallel for schedule(dynamic)
    for (int h = 0; h < H; ++h) {
        std::vector<float> q((size_t)Tn * dh), k((size_t)Tn * dh), vt((size_t)dh * Tn), p(Tn);
        for (int t = 0; t < Tn; ++t) for (int d = 0; d < dh; ++d) {
            const float *r = qkv.data() + (size_t)t * 3 * D + h * dh + d;
            q[(size_t)t * dh + d] = r[0] * scale; k[(size_t)t * dh + d] = r[D]; vt[(size_t)d * Tn + t] = r[2 * D];
        }
        for (int tq = 0; tq < Tn; ++tq) {
            for (int tk = 0; tk < Tn; ++tk) p[tk] = vec_dot_f32(dh, &k[(size_t)tk * dh], &q[(size_t)tq * dh]);
            op_softmax_row(p.data(), Tn);
            for (int d = 0; d < dh; ++d) ctx[(size_t)tq * D + h * dh + d] = vec_dot_f32(Tn, &vt[(size_t)d * Tn], p.data());
        }
    }
    linear(m, pfx + "proj", ctx.data(), Tn, out);
}

// NNSelfAttention::forward (minigpt4.cpp:1095-1244); kv_src = hidden states (self) or encoder states (cross)
static void bert_attention(const Model *m, const std::string &pfx, const float *hidden, int nq, const float *kv_src, int nkv, float *out) {
    const int HID = 768, NH = 12, HD = 64;
    std::vector<float> q((size_t)nq * HID), k((size_t)nkv * HID), vv((size_t)nkv * HID), ctx((size_t)nq * HID);
    linear(m, pfx + "self.key", kv_src, nkv, k.data());
    linear(m, pfx + "self.value", kv_src, nkv, vv.data());
    linear(m, pfx + "self.query", hidden, nq, q.data());
#pragma omp parallel for schedule(dynamic)
    for (int h = 0; h < NH; ++h) {
        std::vector<float> p(nkv), vt((size_t)HD * nkv);
        for (int t = 0; t < nkv; ++t) for (int d = 0; d < HD; ++d) vt[(size_t)d * nkv + t] = vv[(size_t)t * HID + h * HD + d];
        for (int tq = 0; tq < nq; ++tq) {
            for (int tk = 0; tk < nkv; ++tk) p[tk] = vec_dot_f32(HD, &k[(size_t)tk * HID + h * HD], &q[(size_t)tq * HID + h * HD]) / 8.0f;  // sqrt(64)
            // + attention mask: all-zero (self mask uninitialised-zero :2252; encoder mask (1-1)*FLT_MIN = 0 :2263-2268)
            for (int tk = 0; tk < nkv; ++tk) p[tk] = p[tk] + 0.0f;
            op_softmax_row(p.data(), nkv);
            for (int d = 0; d < HD; ++d) ctx[(size_t)tq * HID + h * HD + d] = vec_dot_f32(nkv, &vt[(size_t)d * nkv], p.data());
        }
    }
    std::vector<float> dense((size_t)nq * HID);
    linear(m, pfx + "output.dense", ctx.data(), nq, dense.data());
    for (size_t i = 0; i < dense.size(); ++i) dense[i] += hidden[i];
    op_layernorm(dense.data(), out, HID, nq, F(m, pfx + "output.LayerNorm.weight"), F(m, pfx + "output.LayerNorm.bias"));
}

static int vit_encode(const Model *m, const float *image, float *out, int tap_kind, int tap_idx, float *tap, const VitStages &st) {
    const Tensor &pos = T(m, "visual_encoder.pos_embed");
    VitDims v; v.D = (int)pos.ne[0]; v.T = (int)pos.ne[1]; v.dh = 88; v.H = v.D / 88; v.patch = 14; v.P = 16;
    const int D = v.D, Tn = v.T, IMG = 224;
    v.nblocks = 0; while (Topt(m, "visual_encoder.blocks." + std::to_string(v.nblocks) + ".norm1.weight")) v.nblocks++;

    // patch embed: ggml_conv_2d stride=kernel=14 (minigpt4.cpp:1047-1072): patches -> F16, F16 dot, + bias
    const Tensor &pw = T(m, "visual_encoder.patch_embed.proj.weight");  // F16 ne=[14,14,3,D]
    const float *pb = F(m, "visual_encoder.patch_embed.proj.bias");
    const int KE = 14 * 14 * 3;
    std::vector<float> x((size_t)Tn * D), y((size_t)Tn * D), tmp((size_t)Tn * D);
    {
        std::vector<f16_t> patches((size_t)256 * KE);
        for (int oy = 0; oy < 16; ++oy) for (int ox = 0; ox < 16; ++ox) for (int ic = 0; ic < 3; ++ic) for (int ky = 0; ky < 14; ++ky) for (int kx = 0; kx < 14; ++kx)
            patches[(size_t)(oy * 16 + ox) * KE + ic * 196 + ky * 14 + kx] = f2h(image[(size_t)ic * IMG * IMG + (oy * 14 + ky) * IMG + ox * 14 + kx]);
        const float *cls = F(m, "visual_encoder.cls_token");
        for (int c = 0; c < D; ++c) x[c] = 0.0f + cls[c];
#pragma omp parallel for schedule(static)
        for (int p = 0; p < 256; ++p) for (int oc = 0; oc < D; ++oc)
            x[(size_t)(1 + p) * D + oc] = 0.0f + (pb[oc] + vec_dot_f16(KE, (const f16_t *)pw.data + (size_t)oc * KE, &patches[(size_t)p * KE]));
        const float *pe = (const float *)pos.data;
        for (size_t i = 0; i < (size_t)Tn * D; ++i) x[i] += pe[i];
    }
    if (tap_kind == 1) { memcpy(tap, x.data(), sizeof(float) * Tn * D); return 0; }
    if (st.embed) memcpy(st.embed, x.data(), sizeof(float) * Tn * D);

    std::vector<float> h1((size_t)Tn * 6144 * (D / 1408 + 1));
    for (int b = 0; b < v.nblocks; ++b) {
        const std::string p = "visual_encoder.blocks." + std::to_string(b) + ".";
        op_layernorm(x.data(), y.data(), D, Tn, F(m, p + "norm1.weight"), F(m, p + "norm1.bias"));
        vit_attention(m, p + "attn.", v, y.data(), tmp.data());
        for (size_t i = 0; i < x.size(); ++i) x[i] += tmp[i];
        op_layernorm(x.data(), y.data(), D, Tn, F(m, p + "norm2.weight"), F(m, p + "norm2.bias"));
        const int FF = (int)T(m, p + "mlp.fc1.weight").ne[1];
        h1.resize((size_t)Tn * FF);
        linear(m, p + "mlp.fc1", y.data(), Tn, h1.data());
        for (size_t i = 0; i < h1.size(); ++i) h1[i] = op_gelu(h1[i]);
        linear(m, p + "mlp.fc2", h1.data(), Tn, tmp.data());
        for (size_t i = 0; i < x.size(); ++i) x[i] += tmp[i];
        if (tap_kind == 2 && tap_idx == b) { memcpy(tap, x.data(), sizeof(float) * Tn * D); return 0; }
        if (st.vit_blocks) memcpy(st.vit_blocks + (size_t)b * Tn * D, x.data(), sizeof(float) * Tn * D);
    }
    op_layernorm(x.data(), y.data(), D, Tn, F(m, "ln_vision.weight"), F(m, "ln_vision.bias"));
    const float *image_embeds = y.data();
    if (tap_kind == 3) { memcpy(tap, y.data(), sizeof(float) * Tn * D); return 0; }
    if (st.ln_vision) memcpy(st.ln_vision, y.data(), sizeof(float) * Tn * D);

    // Q-Former (minigpt4.cpp:2203-2340, NNBertEncoderLayer :1324-1463)
    const int NQ = 32, HID = 768;
    std::vector<float> hs((size_t)NQ * HID), a((size_t)NQ * HID), c((size_t)NQ * HID), inter, o((size_t)NQ * HID);
    op_layernorm(F(m, "query_tokens.weight"), hs.data(), HID, NQ, F(m, "Qformer.bert.embeddings.LayerNorm.weight"), F(m, "Qformer.bert.embeddings.LayerNorm.bias"));
    int nl = 0; while (Topt(m, "Qformer.bert.encoder.layer." + std::to_string(nl) + ".attention.self.query.weight")) nl++;
    for (int l = 0; l < nl; ++l) {
        const std::string p = "Qformer.bert.encoder.layer." + std::to_string(l) + ".";
        bert_attention(m, p + "attention.", hs.data(), NQ, hs.data(), NQ, a.data());
        const float *ffn_in = a.data();
        if (Topt(m, p + "crossattention.self.query.weight")) {
            bert_attention(m, p + "crossattention.", a.data(), NQ, image_embeds, Tn, c.data());
            ffn_in = c.data();
        }
        const int FF = (int)T(m, p + "intermediate_query.dense.weight").ne[1];
        inter.resize((size_t)NQ * FF);
        linear(m, p + "intermediate_query.dense", ffn_in, NQ, inter.data());
        for (size_t i = 0; i < inter.size(); ++i) inter[i] = op_gelu(inter[i]);
        linear(m, p + "output_query.dense", inter.data(), NQ, o.data());
        for (size_t i = 0; i < o.size(); ++i) o[i] += ffn_in[i];
        op_layernorm(o.data(), hs.data(), HID, NQ, F(m, p + "output_query.LayerNorm.weight"), F(m, p + "output_query.LayerNorm.bias"));
        if (tap_kind == 4 && tap_idx == l) { memcpy(tap, hs.data(), sizeof(float) * NQ * HID); return 0; }
        if (st.qformer) memcpy(st.qformer + (size_t)l * NQ * HID, hs.data(), sizeof(float) * NQ * HID);
    }
    linear(m, "llama_proj", hs.data(), NQ, out);
    return 0;
}
ORACLE_API int oracle_vit_encode(void *model, const float *image, float *out, int n_threads, int tap_kind, int tap_idx, float *tap) {
    if (n_threads > 0) omp_set_num_threads(n_threads);
    return vit_encode((const Model *)model, image, out, tap_kind, tap_idx, tap, VitStages{nullptr, nullptr, nullptr, nullptr});
}
ORACLE_API int oracle_vit_encode_stages(void *model, const float *image, float *out, int n_threads, float *embed, float *vit_blocks, float *ln_vision,
                                        float *qformer) {
    if (n_threads > 0) omp_set_num_threads(n_threads);
    return vit_encode((const Model *)model, image, out, 0, 0, nullptr, VitStages{embed, vit_blocks, ln_vision, qformer});
}

// ---------------------------------------------------------------------------------------------
// language graph: llama.cpp llama_eval_internal @ master-31cfbb1 (SURVEY §A.3)
// ---------------------------------------------------------------------------------------------
struct Llama {
    const Model *m; int n_vocab, n_embd, n_head, n_layer, n_ff, n_ctx, hd;
    std::vector<f16_t> kc, vc;  // [layer][n_ctx][n_embd] each (V kept token-major; ggml stores it transposed — same values)
    std::vector<float> logits;
};
ORACLE_API void *oracle_llama_new(void *model, int n_ctx) {
    Llama *L = new Llama(); L->m = (const Model *)model;
    const Tensor &te = T(L->m, "tok_embeddings.weight");
    L->n_embd = (int)te.ne[0]; L->n_vocab = (int)te.ne[1];
    L->n_layer = 0; while (Topt(L->m, "layers." + std::to_string(L->n_layer) + ".attention.wq.weight")) L->n_layer++;
    L->n_ff = (int)T(L->m, "layers.0.feed_forward.w1.weight").ne[1];
    L->hd = 128; L->n_head = L->n_embd / L->hd; L->n_ctx = n_ctx;
    L->kc.assign((size_t)L->n_layer * n_ctx * L->n_embd, 0); L->vc.assign((size_t)L->n_layer * n_ctx * L->n_embd, 0);
    L->logits.assign(L->n_vocab, 0.f);
    return L;
}
ORACLE_API void oracle_llama_free(void *l) { delete (Llama *)l; }
ORACLE_API void oracle_llama_set_nhead(void *l, int n_head) { Llama *L = (Llama *)l; L->n_head = n_head; L->hd = L->n_embd / n_head; }

// one head of one row of LLaMA attention over keys 0 .. nvis - 1 of an F16 cache with row stride E (kr / vr point at the head's first
// column); q is rounded to F16 and the soft-max probabilities too (ggml semantics).
// canonical orders = csrc/llama_kernels.cuh attention_head: 16 lanes x 8 dims per key then a 16-lane butterfly;
// soft-max sum: 256 strided double partials + block_sum_256; P.V: 16 key groups (key mod 16), combined by a pairwise tree
static void attention_row(const float *q, const f16_t *kr, const f16_t *vr, int E, int nvis, int hd, float kq_scale, float *out) {
    std::vector<f16_t> qh(hd), ph(nvis); std::vector<float> pr(nvis);
    for (int d = 0; d < hd; ++d) qh[d] = f2h(q[d]);
    for (int t = 0; t < nvis; ++t) {
        const f16_t *k = &kr[(size_t)t * E];
        float lane[16];
        for (int l = 0; l < 16; ++l) { float sacc = 0.f; for (int e = 0; e < 8; ++e) sacc = fmaf(h2f(k[l * 8 + e]), h2f(qh[l * 8 + e]), sacc); lane[l] = sacc; }
        pr[t] = butterfly(lane, 16) * kq_scale;
    }
    float mx = -INFINITY; for (int t = 0; t < nvis; ++t) mx = fmaxf(mx, pr[t]);
    double part[256];
    for (int tt = 0; tt < 256; ++tt) { double sacc = 0; for (int t = tt; t < nvis; t += 256) { const float e = h2f(g_tab_exp[f2h(pr[t] - mx)]); pr[t] = e; sacc += (double)e; } part[tt] = sacc; }
    const float inv = (float)(1.0 / block_sum_256(part));
    for (int t = 0; t < nvis; ++t) ph[t] = f2h(pr[t] * inv);
    for (int d = 0; d < hd; ++d) {
        float g16[16];
        for (int g = 0; g < 16; ++g) g16[g] = 0.f;
        for (int t = 0; t < nvis; ++t) g16[t & 15] = fmaf(h2f(vr[(size_t)t * E + d]), h2f(ph[t]), g16[t & 15]);
        for (int st = 1; st < 16; st <<= 1) for (int g = 0; g < 16; g += 2 * st) g16[g] = g16[g] + g16[g + st];  // pairwise tree
        out[d] = g16[0];
    }
}

// the attention op of the language graph by itself: q F32 [rows][n_head * 128], k / v F16 [n_ctx][n_head * 128], row t at position pos[t]
// (it sees keys 0 .. pos[t]); out F32 [rows][n_head * 128].  Returns 1 on a position outside the cache.
ORACLE_API int oracle_llama_attention(const float *q, const f16_t *k, const f16_t *v, int n_head, int n_ctx, int rows, const int *pos, int n_threads, float *out) {
    for (int t = 0; t < rows; ++t) if (pos[t] < 0 || pos[t] >= n_ctx) return 1;
    if (n_threads > 0) omp_set_num_threads(n_threads);
    const int hd = 128, E = n_head * hd;
    const float kq_scale = 1.0f / sqrtf((float)E / n_head);
#pragma omp parallel for schedule(dynamic) collapse(2)
    for (int h = 0; h < n_head; ++h) for (int t = 0; t < rows; ++t)
        attention_row(&q[(size_t)t * E + h * hd], k + h * hd, v + h * hd, E, pos[t] + 1, hd, kq_scale, &out[(size_t)t * E + h * hd]);
    return 0;
}

// tokens != NULL -> llama_eval; else embd (F32 [N][n_embd]) -> llama_eval_embd.  Keeps last row's logits.
// all_logits (optional): F32 [N][n_vocab] for every row (test aid; the reference keeps only the last).
ORACLE_API int oracle_llama_eval(void *l, const int32_t *tokens, const float *embd, int N, int n_past, int n_threads, float *logits_out, float *hidden_tap, int tap_layer) {
    Llama *L = (Llama *)l; const Model *m = L->m;
    if (n_threads > 0) omp_set_num_threads(n_threads);
    const int E = L->n_embd, H = L->n_head, hd = L->hd, FF = L->n_ff, C = L->n_ctx;
    if (n_past + N > C) return 1;
    std::vector<float> inp((size_t)N * E), cur((size_t)N * E), q((size_t)N * E), k((size_t)N * E), vv((size_t)N * E), att((size_t)N * E), ff1((size_t)N * FF), ff3((size_t)N * FF);
    if (tokens) { const Tensor &te = T(m, "tok_embeddings.weight"); for (int i = 0; i < N; ++i) dequant_row(te, tokens[i], &inp[(size_t)i * E]); }
    else memcpy(inp.data(), embd, sizeof(float) * N * E);
    const float theta_scale = powf(10000.0f, -2.0f / hd);
    const float kq_scale = 1.0f / sqrtf((float)E / H);
    for (int il = 0; il < L->n_layer; ++il) {
        const std::string p = "layers." + std::to_string(il) + ".";
        op_rms_norm_mul(inp.data(), cur.data(), E, N, F(m, p + "attention_norm.weight"));
        mul_mat(T(m, p + "attention.wk.weight"), cur.data(), N, k.data(), true);
        mul_mat(T(m, p + "attention.wq.weight"), cur.data(), N, q.data(), true);
        mul_mat(T(m, p + "attention.wv.weight"), cur.data(), N, vv.data(), true);
        // ggml_rope_inplace mode 0, n_rot = head_dim: adjacent pairs, theta by repeated multiply
        for (int i = 0; i < N; ++i) for (int h = 0; h < H; ++h) {
            float theta = (float)(n_past + i);
            for (int i0 = 0; i0 < hd; i0 += 2) {
                const float c = cosf(theta), s = sinf(theta); theta *= theta_scale;
                float *a = &q[(size_t)i * E + h * hd + i0]; float x0 = a[0], x1 = a[1]; a[0] = x0 * c - x1 * s; a[1] = x0 * s + x1 * c;
                a = &k[(size_t)i * E + h * hd + i0]; x0 = a[0]; x1 = a[1]; a[0] = x0 * c - x1 * s; a[1] = x0 * s + x1 * c;
            }
        }
        f16_t *kc = &L->kc[(size_t)il * C * E], *vc = &L->vc[(size_t)il * C * E];
        for (int i = 0; i < N; ++i) for (int e = 0; e < E; ++e) { kc[(size_t)(n_past + i) * E + e] = f2h(k[(size_t)i * E + e]); vc[(size_t)(n_past + i) * E + e] = f2h(vv[(size_t)i * E + e]); }
#pragma omp parallel for schedule(dynamic) collapse(2)
        for (int h = 0; h < H; ++h) for (int i = 0; i < N; ++i)  // row i sees keys 0 .. n_past + i (ggml_diag_mask_inf masks the rest to -inf -> 0)
            attention_row(&q[(size_t)i * E + h * hd], kc + h * hd, vc + h * hd, E, n_past + i + 1, hd, kq_scale, &att[(size_t)i * E + h * hd]);
        mul_mat(T(m, p + "attention.wo.weight"), att.data(), N, cur.data(), true);
        for (size_t i = 0; i < (size_t)N * E; ++i) inp[i] = cur[i] + inp[i];  // inpFF
        op_rms_norm_mul(inp.data(), cur.data(), E, N, F(m, p + "ffn_norm.weight"));
        mul_mat(T(m, p + "feed_forward.w3.weight"), cur.data(), N, ff3.data(), true);
        mul_mat(T(m, p + "feed_forward.w1.weight"), cur.data(), N, ff1.data(), true);
        for (size_t i = 0; i < (size_t)N * FF; ++i) ff1[i] = op_silu(ff1[i]) * ff3[i];
        mul_mat(T(m, p + "feed_forward.w2.weight"), ff1.data(), N, cur.data(), true);
        for (size_t i = 0; i < (size_t)N * E; ++i) inp[i] = cur[i] + inp[i];
        if (hidden_tap && tap_layer == il) memcpy(hidden_tap, inp.data(), sizeof(float) * N * E);
    }
    op_rms_norm_mul(inp.data(), cur.data(), E, N, F(m, "norm.weight"));
    mul_mat(T(m, "output.weight"), &cur[(size_t)(N - 1) * E], 1, L->logits.data(), true);
    if (logits_out) memcpy(logits_out, L->logits.data(), sizeof(float) * L->n_vocab);
    return 0;
}
ORACLE_API int oracle_llama_n_vocab(void *l) { return ((Llama *)l)->n_vocab; }
ORACLE_API int oracle_llama_n_embd(void *l) { return ((Llama *)l)->n_embd; }
ORACLE_API int oracle_num_threads(void) { return omp_get_max_threads(); }
ORACLE_API void oracle_set_num_threads(int n) { if (n > 0) omp_set_num_threads(n); }

// ---------------------------------------------------------------------------------------------------------------------------
// Host DRAM read bandwidth (bench.py prints it next to the CPU arm: a CPU decode cannot exceed read bandwidth / weight bytes per
// token, BASELINE.md §3).  Streams a buffer much larger than the last-level cache with all threads; returns GB/s of the best pass.
// ---------------------------------------------------------------------------------------------------------------------------
ORACLE_API double oracle_host_read_gbs(long long bytes, int n_threads, int passes) {
    const size_t n = (size_t)bytes / 32;
    __m256i *buf = (__m256i *)aligned_alloc(64, n * 32);
    if (!buf) return 0.0;
    if (n_threads > 0) omp_set_num_threads(n_threads);
#pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)n; ++i) buf[i] = _mm256_set1_epi32((int)i);  // first touch by the reading thread
    double best = 0.0; volatile long long sink = 0;
    for (int p = 0; p < passes; ++p) {
        const double t0 = omp_get_wtime();
        long long tot = 0;
#pragma omp parallel reduction(+ : tot)
        {
            __m256i a0 = _mm256_setzero_si256(), a1 = a0, a2 = a0, a3 = a0;
#pragma omp for schedule(static) nowait
            for (long long i = 0; i < (long long)(n / 4); ++i) {
                a0 = _mm256_add_epi64(a0, _mm256_load_si256(buf + 4 * i)); a1 = _mm256_add_epi64(a1, _mm256_load_si256(buf + 4 * i + 1));
                a2 = _mm256_add_epi64(a2, _mm256_load_si256(buf + 4 * i + 2)); a3 = _mm256_add_epi64(a3, _mm256_load_si256(buf + 4 * i + 3));
            }
            const __m256i s = _mm256_add_epi64(_mm256_add_epi64(a0, a1), _mm256_add_epi64(a2, a3));
            tot += _mm256_extract_epi64(s, 0) + _mm256_extract_epi64(s, 1) + _mm256_extract_epi64(s, 2) + _mm256_extract_epi64(s, 3);
        }
        const double dt = omp_get_wtime() - t0;
        sink += tot;
        if (dt > 0) best = std::max(best, (double)(n * 32) / dt * 1e-9);
    }
    free(buf);
    return best;
}


// llama.cu — host side of the device-resident LLaMA step (see llama.h, llama_kernels.cuh).
#include "llama_kernels.cuh"
#include "llama_mega6.cuh"
#include "llama_prefill.cuh"
#include "llama_sessions.cuh"
#include "llama_sample.cuh"
#include "llama_score.cuh"
#include "llama_state.cuh"
#include "llama_beam.cuh"
#include "llama_logprob.cuh"
#include "llama_penalty.cuh"
#include "tp.h"
#include <stdlib.h>
#include <math.h>
#include <string.h>
#include <algorithm>
#include <limits>

namespace mg4 {
using namespace k;

static size_t g_max_dyn_smem = 0;

// device bytes allocated by this thread through dmalloc: the owned / shared split that minigpt4_b200_session_info reports
static thread_local size_t t_dev_bytes = 0;
template <class T> static void dmalloc(T **p, size_t n) { CUDA_CHECK(cudaMalloc((void **)p, n)); t_dev_bytes += n; }

constexpr int kMaxBatch = LlamaDevice::kMaxBatch;

// Decode steps of more than 8 columns run their layers through the tensor-core prefill GEMM (record_layers' gemm pass with the slot
// table) from this many columns on, on models that have it (pf_ready_); below it, and on every other model, through the per-op matvecs
// in 8-column chunks.  Batches of up to 8 columns always take the per-op matvecs.
// Measured with tools/wide_batch_bench.py (Vicuna-7B Q4_1, n_ctx 512, 1x H100 80GB HBM3 at 700 W), ms per step tensor-core / per-op:
// B 9: 11.24 / 9.21, 12: 11.53 / 10.02, 16: 12.08 / 12.10, 24: 13.17 / 18.07, 32: 14.33 / 24.31, 48: 21.43 / 36.66, 64: 23.90 / 49.38.
constexpr int kWideGemmMin = 16;

// what the contexts of one model share besides the weight pointers each of them holds: the workspace of the batched passes (built by
// the group's first decode_batch or batched flush; decode_batch uses its first kMaxBatch rows), their stream and the batched decode
// step's graphs
struct LlamaGroup {
    size_t weight_bytes = 0;       // the parent's load minus its own context: weights, operand cache, tables, prefill scratch
    size_t batch_bytes = 0;
    unsigned long long fingerprint = 0;   // LlamaDevice::fingerprint
    cudaStream_t stream = nullptr;
    float *x = nullptr, *q = nullptr, *att = nullptr, *act = nullptr;   // [kPrefillMax] rows (act also holds the qkv GEMM's [rows][3 n_embd] output)
    float *last = nullptr;         // [8] the last rows of the contexts that end in a prompt pass
    unsigned char *qact = nullptr;
    DeviceState *state = nullptr;  // the batch's tokens (the decode graph's embed gathers column t from tokens[t], up to 8 columns)
    int *tok = nullptr;            // [kMaxBatch] the tokens of a decode step of more than 8 columns (embed_rows_kernel gathers them)
    SessionSlot *rows = nullptr, *h_rows = nullptr;     // [kPrefillMax] a slot per row of a prompt pass
    SessionSlot *slots = nullptr, *h_slots = nullptr;   // [kMaxBatch] a slot per context: the columns of a decode step, the contexts that end in a prompt pass
    int *ids = nullptr, *h_ids = nullptr;               // [kMaxBatch] their new arg-max ids
    cudaGraphExec_t graph[kMaxBatch + 1] = {};
    int graph_kernels[kMaxBatch + 1] = {};
    smp::TokenTable tokens{};      // every id's text for sample_until's stop rule (built by the group's first call)
    // score_rows (built by the group's first call): every row's logits of a pass, the DeviceState their matvecs' arg-max atomics land in
    // (never read), and the scored entries of a pass (kPrefillMax rows + the first entry of each context) with their results
    float *score_logits = nullptr;
    DeviceState *score_state = nullptr;
    k::ScoreRow *score_rows = nullptr, *h_score_rows = nullptr;
    k::ScoreOut *score_out = nullptr, *h_score_out = nullptr;
    // beam_search (built by the group's first call): the search state and its pinned mirror, each slot's ids and each hypothesis' ids
    // ([2][kMaxBeams][n_ctx]), the first context's logits and DeviceState at the start of a call, the done flags of the last two chunks
    beam::BeamState *beam = nullptr, *h_beam = nullptr;
    int *beam_ids = nullptr;
    float *beam_snap = nullptr;
    DeviceState *beam_snap_state = nullptr;
    int *h_beam_done = nullptr;
    cudaEvent_t beam_ev[2] = {};
    ~LlamaGroup() {
        for (cudaGraphExec_t g : graph) if (g) cudaGraphExecDestroy(g);
        for (void *p : {(void *)beam, (void *)beam_ids, (void *)beam_snap, (void *)beam_snap_state}) if (p) cudaFree(p);
        for (void *p : {(void *)h_beam, (void *)h_beam_done}) if (p) cudaFreeHost(p);
        for (cudaEvent_t e : beam_ev) if (e) cudaEventDestroy(e);
        for (void *p : {(void *)x, (void *)q, (void *)att, (void *)act, (void *)last, (void *)qact, (void *)state, (void *)tok, (void *)rows, (void *)slots, (void *)ids,
                        (void *)tokens.off, (void *)tokens.bytes, (void *)score_logits, (void *)score_state, (void *)score_rows, (void *)score_out})
            if (p) cudaFree(p);
        for (void *p : {(void *)h_rows, (void *)h_slots, (void *)h_ids, (void *)h_score_rows, (void *)h_score_out}) if (p) cudaFreeHost(p);
        if (stream) cudaStreamDestroy(stream);
    }
};

// device sampler (llama_sample.cuh): a context's generator state and mirostat μ, candidate scratch and the ids of a call, in one
// allocation; the generator state and μ (one copy: μ follows the generator) and the ids go through pinned staging
struct SamplerScratch {
    void *dev = nullptr;
    smp::MtState *mt = nullptr;
    MirostatState *mu = nullptr;   // right after the generator (smp::mirostat_state), in the padding before the ids
    int *cons = nullptr;           // the constraint's state (smp::ConsCol::state), after μ
    int *ids = nullptr, *id = nullptr;
    unsigned long long *keys = nullptr;
    float *logit = nullptr, *p = nullptr, *aux = nullptr;
    uint32_t *h_rng = nullptr;   // [625] pinned, then h_mu, then h_cons
    MirostatState *h_mu = nullptr;
    int *h_cons = nullptr;
    int32_t *h_ids = nullptr;    // [n_ids] pinned
    size_t bytes = 0;
    SamplerScratch(int n_vocab, int n_ids) {
        const size_t V = (size_t)n_vocab, P = (size_t)std::max(2, 1 << (int)ceil(log2((double)std::max(2, n_vocab))));
        const size_t o_ids = (sizeof(smp::MtState) + 255) / 256 * 256, o_keys = o_ids + ((size_t)n_ids * 4 + 255) / 256 * 256, o_id = o_keys + P * 8;
        bytes = o_id + 4 * V * 4;
        CUDA_CHECK(cudaMalloc(&dev, bytes));
        unsigned char *b = (unsigned char *)dev;
        static_assert(sizeof(smp::MtState) == 625 * 4 && sizeof(smp::MtState) + sizeof(MirostatState) + 4 <= (sizeof(smp::MtState) + 255) / 256 * 256,
                      "μ and the constraint's state fit before the ids");
        mt = (smp::MtState *)b; mu = (MirostatState *)(b + sizeof(smp::MtState)); ids = (int *)(b + o_ids); keys = (unsigned long long *)(b + o_keys);
        cons = (int *)(mu + 1);
        id = (int *)(b + o_id); logit = (float *)(b + o_id + V * 4); p = (float *)(b + o_id + 2 * V * 4); aux = (float *)(b + o_id + 3 * V * 4);
        CUDA_CHECK(cudaHostAlloc((void **)&h_rng, 625 * 4 + sizeof(MirostatState) + 4, cudaHostAllocDefault));
        h_mu = (MirostatState *)(h_rng + 625);
        h_cons = (int *)(h_mu + 1);
        CUDA_CHECK(cudaHostAlloc((void **)&h_ids, (size_t)n_ids * 4, cudaHostAllocDefault));
    }
    ~SamplerScratch() { if (dev) cudaFree(dev); if (h_rng) cudaFreeHost(h_rng); if (h_ids) cudaFreeHost(h_ids); }
    smp::SampleCtx ctx(const float *logits, DeviceState *state, SessionSlot *slot, int n_past0) const {
        return smp::SampleCtx{logits, state, slot, n_past0, mt, ids, keys, id, logit, p, aux};
    }
};

// sample_until's per-context state (llama_sample.cuh): the ReplyState and the logits snapshot on the device, a pinned mirror of the
// ReplyState, and the done flags and chunk events of the calls this context leads (its column 0)
struct ReplyScratch {
    smp::UntilState *r = nullptr, *h_r = nullptr;
    float *snap = nullptr;
    int *h_done = nullptr;   // [2][kMaxBatch] pinned: the done flags after the last two chunks issued
    cudaEvent_t ev[2] = {};
    size_t bytes = 0;
    explicit ReplyScratch(int n_vocab) {
        bytes = sizeof(smp::UntilState) + (size_t)n_vocab * 4;
        CUDA_CHECK(cudaMalloc((void **)&r, bytes));
        snap = (float *)(r + 1);
        CUDA_CHECK(cudaHostAlloc((void **)&h_r, sizeof(smp::UntilState), cudaHostAllocDefault));
        CUDA_CHECK(cudaHostAlloc((void **)&h_done, 2 * kMaxBatch * sizeof(int), cudaHostAllocDefault));
        for (cudaEvent_t &e : ev) CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    ~ReplyScratch() {
        if (r) cudaFree(r);
        if (h_r) cudaFreeHost(h_r);
        if (h_done) cudaFreeHost(h_done);
        for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    }
};

// sample_until_logprobs' records of one context (llama_logprob.cuh): n_ctx steps on the device and their pinned mirror
struct LogprobScratch {
    lp::Record *rec = nullptr, *h_rec = nullptr;
    size_t bytes = 0;
    explicit LogprobScratch(int n_ctx) {
        bytes = (size_t)n_ctx * sizeof(lp::Record);
        CUDA_CHECK(cudaMalloc((void **)&rec, bytes));
        CUDA_CHECK(cudaHostAlloc((void **)&h_rec, bytes, cudaHostAllocDefault));
    }
    ~LogprobScratch() {
        if (rec) cudaFree(rec);
        if (h_rec) cudaFreeHost(h_rec);
    }
};

// sample_until_penalized's state of one context (llama_penalty.cuh): the penalised row and the window counts (zeroed once; every launch
// leaves them zero), then the history tail on the device and its pinned staging
struct PenaltyScratch {
    float *row = nullptr;
    int *count = nullptr, *tail = nullptr, *h_tail = nullptr;
    int cap = 0;
    size_t bytes = 0;
    PenaltyScratch(int n_vocab, int n_tail) : cap(n_tail) {
        bytes = (size_t)LlamaDevice::kPenaltyBytesPerId * n_vocab + 4 * (size_t)cap;
        CUDA_CHECK(cudaMalloc((void **)&row, bytes));
        count = (int *)(row + n_vocab);
        tail = count + n_vocab;
        CUDA_CHECK(cudaMemset(count, 0, (size_t)n_vocab * 4));
        CUDA_CHECK(cudaHostAlloc((void **)&h_tail, std::max<size_t>(1, (size_t)cap) * 4, cudaHostAllocDefault));
    }
    ~PenaltyScratch() {
        if (row) cudaFree(row);
        if (h_tail) cudaFreeHost(h_tail);
    }
};

// matvec_kernel, or with a slot table matvec_sessions_kernel (per-context positions, caches and logits; llama_sessions.cuh)
template <int WT, int NT>
static void launch_mv(const MatvecArgs &a, const SessionSlot *slots, size_t kv_off, int grid, size_t smem, cudaStream_t s) {
    static bool configured[2][64] = {};   // the attribute is per device (minigpt4_b200_set_device: several contexts of one process may sit on different GPUs)
    int dev = 0; cudaGetDevice(&dev);
    bool &done = configured[slots != nullptr][dev & 63];
    if (!done) {
        const void *fn = slots ? (const void *)matvec_sessions_kernel<WT, NT> : (const void *)matvec_kernel<WT, NT>;
        CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g_max_dyn_smem));
        done = true;
    }
    if (slots) matvec_sessions_kernel<WT, NT><<<grid, kThreads, smem, s>>>(SessionMatvecArgs{a, slots, kv_off});
    else matvec_kernel<WT, NT><<<grid, kThreads, smem, s>>>(a);
}
template <int WT>
static void launch_mv_nt(int nt, const MatvecArgs &a, const SessionSlot *slots, size_t kv_off, int grid, size_t smem, cudaStream_t s) {
    switch (nt) {
        case 1: launch_mv<WT, 1>(a, slots, kv_off, grid, smem, s); break;
        case 2: launch_mv<WT, 2>(a, slots, kv_off, grid, smem, s); break;
        case 4: launch_mv<WT, 4>(a, slots, kv_off, grid, smem, s); break;
        default: launch_mv<WT, 8>(a, slots, kv_off, grid, smem, s); break;
    }
}
static int nt_for(int ntok) { return ntok <= 1 ? 1 : ntok <= 2 ? 2 : ntok <= 4 ? 4 : 8; }
// the fields every matvec of a pass shares
static MatvecArgs mv_args(const QMat &w, int ntok, DeviceState *state, unsigned char *staged, const __half *tab_silu) {
    MatvecArgs a{};
    a.w = w; a.n_valid = w.rows; a.ntok = ntok; a.state = state; a.staged = staged; a.tab_silu = tab_silu;
    return a;
}

static void launch_stage(const MatvecArgs &a, cudaStream_t s, unsigned long long *counter) {
    const int act = act_of(a.w.type);
    const size_t astride = act_bytes(act, a.w.cols);
    switch (act) {
        case ACT_Q8_0: stage_kernel<ACT_Q8_0><<<a.ntok, kThreads, 0, s>>>(a.x, a.x_stride, a.norm_w, a.w.cols, a.staged, astride); break;
        case ACT_Q8_1: stage_kernel<ACT_Q8_1><<<a.ntok, kThreads, 0, s>>>(a.x, a.x_stride, a.norm_w, a.w.cols, a.staged, astride); break;
        case ACT_Q8_K: stage_kernel<ACT_Q8_K><<<a.ntok, kThreads, 0, s>>>(a.x, a.x_stride, a.norm_w, a.w.cols, a.staged, astride); break;
        default: stage_kernel<ACT_F16><<<a.ntok, kThreads, 0, s>>>(a.x, a.x_stride, a.norm_w, a.w.cols, a.staged, astride); break;
    }
    CUDA_CHECK(cudaGetLastError());
    if (counter) ++*counter;
}
// a.ntok (<= 8) rows through one matrix; slots / kv_off: matvec_sessions_kernel (EPI_QKV / EPI_LOGITS into each row's own context).
// restage = false when the previous launch staged the same input in the same format (unfused q/k/v of one type)
static void launch_matvec(MatvecArgs a, int sm_count, cudaStream_t s, unsigned long long *counter, const SessionSlot *slots = nullptr, size_t kv_off = 0,
                          bool restage = true) {
    if (restage) launch_stage(a, s, counter);
    const int rows = a.w.rows, nt = nt_for(a.ntok);
    const int target = 2 * sm_count * kWarps;
    int rpw = (rows + target - 1) / target;
    rpw = std::max(2, (rpw + 1) & ~1);
    a.rows_per_warp = rpw;
    const int grid = (rows + kWarps * rpw - 1) / (kWarps * rpw);
    const size_t smem = (size_t)nt * act_bytes(act_of(a.w.type), a.w.cols);
    if (smem > g_max_dyn_smem) MG4_PANIC("activation staging needs %zu B of shared memory (> %zu)", smem, g_max_dyn_smem);
    switch (a.w.type) {
        case GG_Q4_0: launch_mv_nt<GG_Q4_0>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q4_1: launch_mv_nt<GG_Q4_1>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q5_K: launch_mv_nt<GG_Q5_K>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q4_K: launch_mv_nt<GG_Q4_K>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q5_0: launch_mv_nt<GG_Q5_0>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q5_1: launch_mv_nt<GG_Q5_1>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q8_0: launch_mv_nt<GG_Q8_0>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_Q6_K: launch_mv_nt<GG_Q6_K>(nt, a, slots, kv_off, grid, smem, s); break;
        case GG_F16: launch_mv_nt<GG_F16>(nt, a, slots, kv_off, grid, smem, s); break;
        default: MG4_PANIC("no matvec kernel for ggml type %d", a.w.type);
    }
    CUDA_CHECK(cudaGetLastError());
    if (counter) ++*counter;
}

// attention scratch = n_ctx * 6 bytes of dynamic shared memory.  The attribute is per device and kernel, and it only grows: contexts of one
// process may differ in n_ctx, and lowering it would make every later attention launch of a context with a larger n_ctx fail.
static void attn_smem(int n_ctx) {
    static int set[2][64] = {};
    int dev = 0; CUDA_CHECK(cudaGetDevice(&dev));
    const int need = std::max(49152, n_ctx * 6);
    const void *fn[2] = {(const void *)attn_kernel, (const void *)attn_sessions_kernel};
    for (int k = 0; k < 2; ++k)
        if (need > set[k][dev & 63]) { CUDA_CHECK(cudaFuncSetAttribute(fn[k], cudaFuncAttributeMaxDynamicSharedMemorySize, need)); set[k][dev & 63] = need; }
}

// ------------------------------------------------------------------------------------------------
// weight upload + repack
// ------------------------------------------------------------------------------------------------
static bool type_supported(int t) {  // (Q4_K, Q5_0, Q5_1, Q8_0: tests/test_block_types_gpu.py)
    return t == GG_Q4_0 || t == GG_Q4_1 || t == GG_Q4_K || t == GG_Q5_K || t == GG_Q6_K || t == GG_F16 || t == GG_Q5_0 || t == GG_Q5_1 || t == GG_Q8_0;
}

static void qmat_alloc(QMat &m, int type, int rows, int cols) {
    m.type = type; m.rows = (rows + 1) & ~1; m.cols = cols;
    const size_t R = (size_t)m.rows;
    auto zalloc = [](void **p, size_t n) { dmalloc(p, n); CUDA_CHECK(cudaMemset(*p, 0, n)); };
    switch (type) {
        case GG_Q4_0: m.row_bytes = (cols / 32 * 18 + 15) & ~15; zalloc(&m.p0, R * m.row_bytes + 256); break;
        case GG_Q4_1: m.row_bytes = (cols / 32 * 20 + 15) & ~15; zalloc(&m.p0, R * m.row_bytes + 256); break;
        case GG_Q5_K: m.row_bytes = cols / 256 * 176; zalloc(&m.p0, R * m.row_bytes + 256); break;   // row-packed: [nsb x 128 B qs][nsb x 32 B qh][nsb x 16 B scales, d, dmin]
        case GG_Q4_K: zalloc(&m.p0, R * cols / 256 * 128); zalloc(&m.p2, R * cols / 256 * 16); break;
        case GG_Q8_0: zalloc(&m.p0, R * cols / 32 * 32); zalloc(&m.p2, R * cols / 32 * 2); break;
        case GG_Q5_0: zalloc(&m.p0, R * cols / 32 * 16); zalloc(&m.p1, R * cols / 32 * 4); zalloc(&m.p2, R * cols / 32 * 2); break;
        case GG_Q5_1: zalloc(&m.p0, R * cols / 32 * 16); zalloc(&m.p1, R * cols / 32 * 4); zalloc(&m.p2, R * cols / 32 * 4); break;
        case GG_Q6_K: zalloc(&m.p0, R * cols / 256 * 128); zalloc(&m.p1, R * cols / 256 * 64); zalloc(&m.p2, R * cols / 256 * 16); zalloc(&m.p3, R * cols / 256 * 2); break;
        case GG_F16: zalloc(&m.p0, R * cols * 2); break;
        default: MG4_PANIC("unsupported weight type %d", type);
    }
    m.bytes = (size_t)rows * gg_row_bytes(type, (size_t)cols);
}
static void qmat_free(QMat &m) {
    for (void **p : {&m.p0, &m.p1, &m.p2, &m.p3}) if (*p) { cudaFree(*p); *p = nullptr; }
}

struct Stager {  // raw tensor bytes -> device scratch
    unsigned char *dev = nullptr; size_t cap = 0;
    unsigned char *put(const void *host, size_t n) {
        if (n > cap) { if (dev) cudaFree(dev); cap = n + (n >> 2); CUDA_CHECK(cudaMalloc((void **)&dev, cap)); }
        CUDA_CHECK(cudaMemcpy(dev, host, n, cudaMemcpyHostToDevice));
        return dev;
    }
    ~Stager() { if (dev) cudaFree(dev); }
};

// copy rows [row0,row0+nrows) x column range [col0,col0+ncols) of src into dst at dst_row = r*row_mul + row_off, dst_col0
static void repack_into(QMat &dst, const HostTensor &src, Stager &st, int row0, int nrows, int col0, int ncols, int row_mul, int row_off, int dst_col0) {
    const int src_cols = (int)src.ne[0];
    const size_t rb = gg_row_bytes(src.gg, (size_t)src_cols);
    const unsigned char *raw = st.put(src.data + (size_t)row0 * rb, (size_t)nrows * rb);
    const int be = (int)gg_block_elems(src.gg);
    const int src_nb = src_cols / be, blk0 = col0 / be, nblk = ncols / be, dst_nb = dst.cols / be, dblk0 = dst_col0 / be;
    const size_t n = (size_t)nrows * nblk;
    const int th = 256; const unsigned gr = (unsigned)((n + th - 1) / th);
    switch (src.gg) {
        case GG_Q4_0: repack_q4<<<gr, th>>>(raw, src_nb, blk0, nblk, nrows, false, (unsigned char *)dst.p0, dst_nb, dst.row_bytes, row_mul, row_off, dblk0); break;
        case GG_Q4_1: repack_q4<<<gr, th>>>(raw, src_nb, blk0, nblk, nrows, true, (unsigned char *)dst.p0, dst_nb, dst.row_bytes, row_mul, row_off, dblk0); break;
        case GG_Q5_K: repack_q5k<<<gr, th>>>(raw, src_nb, blk0, nblk, nrows, (unsigned char *)dst.p0, dst_nb, dst.row_bytes, row_mul, row_off, dblk0); break;
        case GG_Q4_K: repack_q4k<<<gr, th>>>(raw, src_nb, blk0, nblk, nrows, (unsigned char *)dst.p0, (unsigned char *)dst.p2, dst_nb, row_mul, row_off, dblk0); break;
        case GG_Q5_0: case GG_Q5_1: case GG_Q8_0:
            repack_b32<<<gr, th>>>(src.gg, raw, src_nb, blk0, nblk, nrows, (unsigned char *)dst.p0, (unsigned char *)dst.p1, (unsigned char *)dst.p2, dst_nb, row_mul, row_off, dblk0); break;
        case GG_Q6_K: repack_q6k<<<gr, th>>>(raw, src_nb, blk0, nblk, nrows, (unsigned char *)dst.p0, (unsigned char *)dst.p1, (unsigned char *)dst.p2, (unsigned short *)dst.p3, dst_nb, row_mul, row_off, dblk0); break;
        case GG_F16: repack_f16<<<gr, th>>>((const unsigned short *)raw, src_cols, col0, ncols, nrows, (unsigned short *)dst.p0, dst.cols, row_mul, row_off, dst_col0); break;
        default: MG4_PANIC("unsupported weight type %d", src.gg);
    }
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaDeviceSynchronize());  // the stager is reused by the next tensor
}

static float *upload_f32(const HostTensor &t) {
    if (t.gg != GG_F32) MG4_PANIC("tensor %s must be F32", t.name.c_str());
    float *d; dmalloc(&d, t.nbytes); CUDA_CHECK(cudaMemcpy(d, t.data, t.nbytes, cudaMemcpyHostToDevice));
    return d;
}

// ------------------------------------------------------------------------------------------------
LlamaDevice::LlamaDevice() {}
LlamaDevice::~LlamaDevice() {
    if (graph_) cudaGraphExecDestroy(graph_);
    for (void *p : {(void *)kcache_, (void *)vcache_, (void *)x_, (void *)q_, (void *)att_, (void *)act_, (void *)logits_, (void *)partial_, (void *)qact_, (void *)state_})
        if (p) cudaFree(p);
    if (!group_ || group_.use_count() == 1) free_weights();   // (a failed load frees what it got to)
    if (mega_barrier_) cudaFree(mega_barrier_);
    if (mega_trace_) cudaFree(mega_trace_);
    delete (mk6::Params6 *)mega6_params_;
    if (h_state_) cudaFreeHost(h_state_);
    if (h_argmax_) cudaFreeHost(h_argmax_);
    if (ev0_) cudaEventDestroy(ev0_);
    if (ev1_) cudaEventDestroy(ev1_);
    if (stream_) cudaStreamDestroy(stream_);
    smp_.reset();
    reply_.reset();
    logprob_.reset();
    pen_.reset();
}
void LlamaDevice::free_weights() {
    for (auto &L : layers_) { qmat_free(L.qkv); qmat_free(L.wq); qmat_free(L.wk); qmat_free(L.wv); qmat_free(L.wo); qmat_free(L.w13); qmat_free(L.w2); cudaFree(L.attn_norm); cudaFree(L.ffn_norm); }
    qmat_free(output_);
    for (void *p : {(void *)final_norm_, tok_raw_, (void *)rope_, (void *)tab_exp_, (void *)tab_silu_, (void *)embd_in_}) if (p) cudaFree(p);
    for (auto &L : layers_) for (PQMat *m : {&L.pqkv, &L.pwo, &L.pw13, &L.pw2}) { if (m->q) cudaFree(m->q); if (m->sc) cudaFree(m->sc); }
    for (void *p : {(void *)pf_q8_, pf_sc_, (void *)tok_ids_, pf_part_}) if (p) cudaFree(p);
}

static inline unsigned short f2h_bits(float f) { __half h = __float2half_rn(f); unsigned short u; memcpy(&u, &h, 2); return u; }
static inline float h2f_bits(unsigned short u) { __half h; memcpy(&h, &u, 2); return __half2float(h); }
// ggml's fp16 lookup tables of exp and silu (ggml_init), [65536] each, indexed by the F16 bits of the argument
static void fp16_tables(unsigned short *te, unsigned short *ts) {
    for (int i = 0; i < 65536; ++i) { const float x = h2f_bits((unsigned short)i); te[i] = f2h_bits(expf(x)); ts[i] = f2h_bits(x / (1.0f + expf(-x))); }
}

// FNV-1a 64 over the tensor table in name order (name, type, dims) and the first 4096 bytes of every tensor: two files of one spec written
// from different weights differ, and reading it touches a few pages per tensor
static unsigned long long model_fingerprint(const LlamaFile &f) {
    unsigned long long h = 0xcbf29ce484222325ull;
    auto mix = [&h](const void *p, size_t n) { const unsigned char *b = (const unsigned char *)p; for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 0x100000001b3ull; } };
    for (const auto &kv : f.tensors) {
        const HostTensor &t = kv.second;
        mix(t.name.data(), t.name.size());
        const int32_t gg = t.gg;
        mix(&gg, 4);
        mix(t.ne, (size_t)t.n_dims * sizeof(int64_t));
        mix(t.data, std::min<size_t>(t.nbytes, 4096));
    }
    return h;
}

bool LlamaDevice::load(const LlamaFile &f, int n_ctx, TPLink *tp) {
    tp_ = tp;
    const int world = tp ? tp->world : 1, rank = tp ? tp->rank : 0;
    d_.n_vocab = (int)f.n_vocab; d_.n_embd = (int)f.n_embd; d_.n_head = (int)f.n_head; d_.n_layer = (int)f.n_layer;
    d_.n_ff = (int)f.n_ff(); d_.n_ctx = n_ctx; d_.head_dim = d_.n_embd / d_.n_head;
    if (d_.head_dim != 128 || (int)f.n_rot != 128) { MG4_ERR("only head_dim 128 LLaMA models are supported (got %d)", d_.head_dim); return false; }
    if (n_ctx < 8 || n_ctx > 32768) { MG4_ERR("n_ctx %d is outside the supported range 8 .. 32768 (attention scratch = 6 n_ctx bytes of shared memory)", n_ctx); return false; }
    if (d_.n_head % world || d_.n_ff % (32 * world)) { MG4_ERR("tensor-parallel degree %d does not divide the model", world); return false; }
    n_head_local_ = d_.n_head / world; n_embd_local_ = n_head_local_ * 128; n_ff_local_ = d_.n_ff / world;
    const int E = d_.n_embd, El = n_embd_local_, FF = d_.n_ff, FFl = n_ff_local_;

    int dev = 0; CUDA_CHECK(cudaGetDevice(&dev));
    cudaDeviceProp prop; CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    sm_count_ = prop.multiProcessorCount;
    g_max_dyn_smem = std::min<size_t>(prop.sharedMemPerBlockOptin, 220 * 1024) - 1024;
    group_ = std::make_shared<LlamaGroup>();
    group_->fingerprint = model_fingerprint(f);
    const size_t bytes0 = t_dev_bytes;

    Stager st;
    bytes_per_token_ = 0;
    layers_.resize((size_t)d_.n_layer);
    for (int il = 0; il < d_.n_layer; ++il) {
        Layer &L = layers_[(size_t)il];
        const std::string p = "layers." + std::to_string(il) + ".";
        const HostTensor &wq = f.get(p + "attention.wq.weight"), &wk = f.get(p + "attention.wk.weight"), &wv = f.get(p + "attention.wv.weight");
        const HostTensor &wo = f.get(p + "attention.wo.weight");
        const HostTensor &w1 = f.get(p + "feed_forward.w1.weight"), &w2 = f.get(p + "feed_forward.w2.weight"), &w3 = f.get(p + "feed_forward.w3.weight");
        for (const HostTensor *t : {&wq, &wk, &wv, &wo, &w1, &w2, &w3}) {
            if (!type_supported(t->gg)) { MG4_ERR("tensor %s has unsupported type %d", t->name.c_str(), t->gg); return false; }
            const int be = (int)gg_block_elems(t->gg);
            if (world > 1 && be > 1 && ((El % be) || (FFl % be))) { MG4_ERR("tensor-parallel split of %s is not aligned to its %d-element quant blocks", t->name.c_str(), be); return false; }
        }
        if (wq.ne[0] != E || wq.ne[1] != E || w1.ne[1] != FF || w2.ne[0] != FF) { MG4_ERR("unexpected tensor shapes in layer %d", il); return false; }
        if (w1.gg != w3.gg) { MG4_ERR("w1/w3 of layer %d differ in type", il); return false; }
        L.fused_qkv = wq.gg == wk.gg && wk.gg == wv.gg;
        if (L.fused_qkv) {
            qmat_alloc(L.qkv, wq.gg, 3 * El, E);
            repack_into(L.qkv, wq, st, rank * El, El, 0, E, 1, 0, 0);
            repack_into(L.qkv, wk, st, rank * El, El, 0, E, 1, El, 0);
            repack_into(L.qkv, wv, st, rank * El, El, 0, E, 1, 2 * El, 0);
            bytes_per_token_ += L.qkv.bytes;
        } else {
            qmat_alloc(L.wq, wq.gg, El, E); repack_into(L.wq, wq, st, rank * El, El, 0, E, 1, 0, 0);
            qmat_alloc(L.wk, wk.gg, El, E); repack_into(L.wk, wk, st, rank * El, El, 0, E, 1, 0, 0);
            qmat_alloc(L.wv, wv.gg, El, E); repack_into(L.wv, wv, st, rank * El, El, 0, E, 1, 0, 0);
            bytes_per_token_ += L.wq.bytes + L.wk.bytes + L.wv.bytes;
        }
        qmat_alloc(L.wo, wo.gg, E, El); repack_into(L.wo, wo, st, 0, E, rank * El, El, 1, 0, 0);
        qmat_alloc(L.w13, w1.gg, 2 * FFl, E);
        repack_into(L.w13, w1, st, rank * FFl, FFl, 0, E, 2, 0, 0);
        repack_into(L.w13, w3, st, rank * FFl, FFl, 0, E, 2, 1, 0);
        qmat_alloc(L.w2, w2.gg, E, FFl); repack_into(L.w2, w2, st, 0, E, rank * FFl, FFl, 1, 0, 0);
        bytes_per_token_ += L.wo.bytes + L.w13.bytes + L.w2.bytes;
        L.attn_norm = upload_f32(f.get(p + "attention_norm.weight"));
        L.ffn_norm = upload_f32(f.get(p + "ffn_norm.weight"));
    }
    {
        const HostTensor &out = f.get("output.weight");
        if (!type_supported(out.gg)) { MG4_ERR("output.weight has unsupported type %d", out.gg); return false; }
        qmat_alloc(output_, out.gg, d_.n_vocab, E);
        repack_into(output_, out, st, 0, d_.n_vocab, 0, E, 1, 0, 0);
        bytes_per_token_ += output_.bytes;
        final_norm_ = upload_f32(f.get("norm.weight"));
        const HostTensor &tok = f.get("tok_embeddings.weight");
        tok_type_ = tok.gg;
        if (!(type_supported(tok.gg) || tok.gg == GG_F32)) { MG4_ERR("tok_embeddings has unsupported type %d", tok.gg); return false; }
        dmalloc(&tok_raw_, tok.nbytes);
        CUDA_CHECK(cudaMemcpy(tok_raw_, tok.data, tok.nbytes, cudaMemcpyHostToDevice));
    }
    // ggml's fp16 lookup tables (ggml_init): exp and silu, computed with the host libm exactly as ggml does
    {
        std::vector<unsigned short> te(65536), ts(65536);
        fp16_tables(te.data(), ts.data());
        dmalloc(&tab_exp_, 131072); CUDA_CHECK(cudaMemcpy(tab_exp_, te.data(), 131072, cudaMemcpyHostToDevice));
        dmalloc(&tab_silu_, 131072); CUDA_CHECK(cudaMemcpy(tab_silu_, ts.data(), 131072, cudaMemcpyHostToDevice));
    }
    // RoPE table, mode 0: theta_i = pos * 10000^(-2i/n_rot) formed by repeated multiplication, cosf/sinf from libm (ggml_rope_f32)
    {
        const int hd2 = 64;
        std::vector<float2> tab((size_t)n_ctx * hd2);
        const float theta_scale = powf(10000.0f, -2.0f / 128.0f);
        for (int p = 0; p < n_ctx; ++p) { float theta = (float)p; for (int i = 0; i < hd2; ++i) { tab[(size_t)p * hd2 + i] = make_float2(cosf(theta), sinf(theta)); theta *= theta_scale; } }
        dmalloc(&rope_, tab.size() * sizeof(float2));
        CUDA_CHECK(cudaMemcpy(rope_, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice));
    }
    alloc_context();
    // scratch of the synchronous prefill path (eval_rows ends with a stream sync), shared by the sessions of this model
    const size_t R = (size_t)kPrefillMax;
    dmalloc(&tok_ids_, R * 4);
    dmalloc(&embd_in_, (size_t)512 * E * 4);
    CUDA_CHECK(cudaDeviceSynchronize());
    if (tp_ && tp_->world > 1) tp_->setup_peers(E, stream_);
    pf_ready_ = build_prefill();
    { const size_t b = t_dev_bytes; build_graph(); owned_bytes_ += t_dev_bytes - b; }
    group_->weight_bytes = t_dev_bytes - bytes0 - owned_bytes_;
    MG4_INFO("LLaMA on device: %d layers, n_embd %d, n_ff %d, vocab %d, %.1f MB streamed per token, tp %d/%d", d_.n_layer, E, FF, d_.n_vocab,
             bytes_per_token_ / 1048576.0, rank, world);
    return true;
}

void LlamaDevice::alloc_context() {
    const size_t b0 = t_dev_bytes;
    const int E = d_.n_embd, El = n_embd_local_, FF = d_.n_ff, FFl = n_ff_local_;
    CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    CUDA_CHECK(cudaEventCreate(&ev0_)); CUDA_CHECK(cudaEventCreate(&ev1_));
    attn_smem(d_.n_ctx);
    const size_t kv = (size_t)d_.n_layer * d_.n_ctx * El;
    dmalloc(&kcache_, kv * 2); CUDA_CHECK(cudaMemset(kcache_, 0, kv * 2));
    dmalloc(&vcache_, kv * 2); CUDA_CHECK(cudaMemset(vcache_, 0, kv * 2));
    const size_t R = (size_t)kPrefillMax;  // rows of one prefill pass (the per-op path uses the first 8)
    dmalloc(&x_, R * E * 4);
    dmalloc(&q_, R * El * 4);
    dmalloc(&att_, R * El * 4);
    dmalloc(&act_, R * FFl * 4);
    dmalloc(&partial_, (size_t)8 * E * 4);
    dmalloc(&qact_, (size_t)8 * ((size_t)std::max(E, FF) * 2 + 4096));
    dmalloc(&logits_, (size_t)(d_.n_vocab + 1) * 4);
    dmalloc(&state_, sizeof(DeviceState)); CUDA_CHECK(cudaMemset(state_, 0, sizeof(DeviceState)));
    CUDA_CHECK(cudaHostAlloc((void **)&h_state_, sizeof(DeviceState), cudaHostAllocDefault)); memset(h_state_, 0, sizeof(DeviceState));
    CUDA_CHECK(cudaHostAlloc((void **)&h_argmax_, 64, cudaHostAllocDefault)); *h_argmax_ = 0;
    owned_bytes_ += t_dev_bytes - b0;
}

bool LlamaDevice::load_session(const LlamaDevice &p) {
    if (p.tp_ && p.tp_->world > 1) { MG4_ERR("sessions of a tensor-parallel context are not supported"); return false; }
    group_ = p.group_;
    d_ = p.d_; n_head_local_ = p.n_head_local_; n_embd_local_ = p.n_embd_local_; n_ff_local_ = p.n_ff_local_;
    layers_ = p.layers_; output_ = p.output_; final_norm_ = p.final_norm_; tok_raw_ = p.tok_raw_; tok_type_ = p.tok_type_;
    rope_ = p.rope_; tab_exp_ = p.tab_exp_; tab_silu_ = p.tab_silu_; embd_in_ = p.embd_in_; tok_ids_ = p.tok_ids_;
    pf_ready_ = p.pf_ready_; pf_S_e_ = p.pf_S_e_; pf_S_ff_ = p.pf_S_ff_; pf_q8_ = p.pf_q8_; pf_sc_ = p.pf_sc_; pf_part_ = p.pf_part_; pf_part_bytes_ = p.pf_part_bytes_;
    memcpy(pf_tmB_e_, p.pf_tmB_e_, 128); memcpy(pf_tmS_e_, p.pf_tmS_e_, 128); memcpy(pf_tmB_ff_, p.pf_tmB_ff_, 128); memcpy(pf_tmS_ff_, p.pf_tmS_ff_, 128);
    bytes_per_token_ = p.bytes_per_token_; sm_count_ = p.sm_count_;
    alloc_context();
    CUDA_CHECK(cudaDeviceSynchronize());
    { const size_t b = t_dev_bytes; build_graph(); owned_bytes_ += t_dev_bytes - b; }
    MG4_INFO("LLaMA session: %d contexts share %.1f MB of weights, %.1f MB of its own", group_size(), group_->weight_bytes / 1048576.0, owned_bytes_ / 1048576.0);
    return true;
}
size_t LlamaDevice::shared_bytes() const { return group_ ? group_->weight_bytes + group_->batch_bytes : 0; }

// ------------------------------------------------------------------------------------------------
// one pass of all layers over p.rows rows that sit in p.x: every caller (decode graph, prompt passes, the batched decode step and the
// batched prompt pass) records its layers here
// ------------------------------------------------------------------------------------------------
void LlamaDevice::record_layers(const Pass &p) {
    const int E = d_.n_embd, El = n_embd_local_, FFl = n_ff_local_, C = d_.n_ctx;
    const float kq_scale = 1.0f / sqrtf((float)d_.n_embd / (float)d_.n_head);
    if (!p.slots && !p.gemm && p.rows > 8) MG4_PANIC("a per-op pass without a slot table takes at most 8 rows (got %d)", p.rows);  // (positions n_past + t of one launch)
    auto mv = [&](const QMat &w, int m) { return mv_args(w, m, p.state, p.qact, tab_silu_); };
    for (int il = 0; il < d_.n_layer; ++il) {
        Layer &L = layers_[(size_t)il];
        const size_t kv_off = (size_t)il * C * El;
        // qkv: RoPE, and the F16 K / V rows appended at each row's position
        if (p.gemm) {
            pf_stage(L.qkv, p.x, E, L.attn_norm, pf_S_e_, p);
            pf::PrefillArgs a{};
            if (p.slots) { a.epi = EPI_PLAIN; a.out = p.act; a.out_stride = 3 * El; }
            else { a.epi = EPI_QKV; a.q_out = p.q; a.kcache = kcache_ + kv_off; a.vcache = vcache_ + kv_off; a.rope = rope_; a.e_local = El; a.half_dim = 64; }
            pf_gemm(L.pqkv, false, a, p);
            if (p.slots) {
                qkv_rows_kernel<<<dim3((unsigned)((3 * El / 2 + 255) / 256), (unsigned)p.rows), 256, 0, p.s>>>(p.act, p.slots, kv_off, p.q, rope_, El, 64);
                ++*p.counter;
            }
        } else {
            for (int t0 = 0; t0 < p.rows; t0 += 8) {
                MatvecArgs a = mv(L.qkv, std::min(8, p.rows - t0));
                a.x = p.x + (size_t)t0 * E; a.x_stride = E; a.norm_w = L.attn_norm; a.epi = EPI_QKV;
                a.q_out = p.q + (size_t)t0 * El; a.rope = rope_; a.e_local = El; a.half_dim = 64;
                if (!p.slots) { a.kcache = kcache_ + kv_off; a.vcache = vcache_ + kv_off; }
                const SessionSlot *sl = p.slots ? p.slots + t0 : nullptr;
                if (L.fused_qkv) { a.part = -1; launch_matvec(a, sm_count_, p.s, p.counter, sl, kv_off); }
                else {
                    const QMat *ms[3] = {&L.wq, &L.wk, &L.wv};
                    for (int part = 0; part < 3; ++part) {
                        const bool same = part > 0 && act_of(ms[part]->type) == act_of(ms[part - 1]->type);
                        a.w = *ms[part]; a.part = part; a.n_valid = a.w.rows;
                        launch_matvec(a, sm_count_, p.s, p.counter, sl, kv_off, !same);
                    }
                }
            }
        }
        const dim3 ag((unsigned)n_head_local_, (unsigned)p.rows);
        if (p.slots) attn_sessions_kernel<<<ag, 256, (size_t)C * 6, p.s>>>(p.q, p.slots, kv_off, p.att, El, C, kq_scale, tab_exp_);
        else attn_kernel<<<ag, 256, (size_t)C * 6, p.s>>>(p.q, kcache_ + kv_off, vcache_ + kv_off, p.att, p.state, El, C, kq_scale, tab_exp_);
        CUDA_CHECK(cudaGetLastError()); ++*p.counter;
        // wo, gate/up, down
        if (p.gemm) {
            pf_stage(L.wo, p.att, El, nullptr, pf_S_e_, p);
            { pf::PrefillArgs a{}; a.epi = EPI_RESID; a.out = p.x; a.out_stride = E; a.resid = p.x; pf_gemm(L.pwo, false, a, p); }
            pf_stage(L.w13, p.x, E, L.ffn_norm, pf_S_e_, p);
            { pf::PrefillArgs a{}; a.epi = EPI_SWIGLU; a.out = p.act; a.out_stride = FFl; pf_gemm(L.pw13, false, a, p); }
            pf_stage(L.w2, p.act, FFl, nullptr, pf_S_ff_, p);
            { pf::PrefillArgs a{}; a.epi = EPI_RESID; a.out = p.x; a.out_stride = E; a.resid = p.x; pf_gemm(L.pw2, true, a, p); }
        } else {
            for (int t0 = 0; t0 < p.rows; t0 += 8) {
                const int m = std::min(8, p.rows - t0);
                float *x = p.x + (size_t)t0 * E, *act = p.act + (size_t)t0 * FFl;
                MatvecArgs b = mv(L.wo, m);
                b.x = p.att + (size_t)t0 * El; b.x_stride = El;
                add_matvec(b, x, p);
                MatvecArgs g = mv(L.w13, m);
                g.x = x; g.x_stride = E; g.norm_w = L.ffn_norm; g.epi = EPI_SWIGLU; g.out = act; g.out_stride = FFl;
                launch_matvec(g, sm_count_, p.s, p.counter);
                MatvecArgs e = mv(L.w2, m);
                e.x = act; e.x_stride = FFl;
                add_matvec(e, x, p);
            }
        }
    }
    CUDA_CHECK(cudaGetLastError());
}

// wo / down: the product added into the residual rows x.  A tensor-parallel rank adds the sum of every rank's partial product: one kernel
// over peer memory (signal, wait, sum, residual), or NCCL and an add.
void LlamaDevice::add_matvec(MatvecArgs a, float *x, const Pass &p) {
    const int E = d_.n_embd;
    const size_t n = (size_t)a.ntok * E;
    a.out_stride = E;
    if (!tp_ || tp_->world <= 1) { a.epi = EPI_RESID; a.out = x; a.resid = x; launch_matvec(a, sm_count_, p.s, p.counter); }
    else if (tp_->peers_ready()) {
        a.epi = EPI_PLAIN; a.out = tp_->partial_out(); launch_matvec(a, sm_count_, p.s, p.counter);
        tp_->all_reduce_resid(x, x, n, p.s); ++*p.counter;
    } else {
        a.epi = EPI_PLAIN; a.out = partial_; launch_matvec(a, sm_count_, p.s, p.counter);
        tp_->all_reduce_sum(partial_, n, p.s);
        add_kernel<<<(unsigned)((n + 255) / 256), 256, 0, p.s>>>(x, partial_, (int)n); ++*p.counter;
    }
}

// one pass of this context over n rows that sit in x_ at positions state_->n_past + t, then (want_logits) the logits and arg-max of the
// last row, finalize (n_past += n) and the 4-byte arg-max to pinned memory (valid after the next stream sync)
void LlamaDevice::record_pass(int n, bool want_logits) {
    record_layers(Pass{n, x_, q_, att_, act_, qact_, state_, nullptr, pf_ready_ && n >= 2, stream_, &launches_});
    if (want_logits) {
        MatvecArgs o = mv_args(output_, 1, state_, qact_, tab_silu_);
        o.x = x_ + (size_t)(n - 1) * d_.n_embd; o.x_stride = d_.n_embd; o.norm_w = final_norm_; o.epi = EPI_LOGITS; o.out = logits_; o.n_valid = d_.n_vocab;
        launch_matvec(o, sm_count_, stream_, &launches_);
    }
    finalize_kernel<<<1, 32, 0, stream_>>>(state_, want_logits ? 1 : 0, nullptr); ++launches_;
    CUDA_CHECK(cudaGetLastError());
    if (want_logits) CUDA_CHECK(cudaMemcpyAsync(h_argmax_, &state_->argmax_id, 4, cudaMemcpyDeviceToHost, stream_));
}

// the token-embedding rows of the decode graphs: row t gathers DeviceState::tokens[t]
void LlamaDevice::launch_embed(int n, const DeviceState *st, float *x, cudaStream_t s, unsigned long long *counter) const {
    const unsigned char *tok = (const unsigned char *)tok_raw_;
    const size_t rb = gg_row_bytes(tok_type_, (size_t)d_.n_embd);
    if (tok_type_ == GG_Q4_K) embed_q4k_kernel<<<n, 256, 0, s>>>(tok, rb, d_.n_embd, st, x);
    else if (tok_type_ == GG_Q5_0 || tok_type_ == GG_Q5_1 || tok_type_ == GG_Q8_0) embed_b32_kernel<<<n, 256, 0, s>>>(tok_type_, tok, rb, d_.n_embd, st, x);
    else embed_kernel<<<n, 256, 0, s>>>(tok_type_, tok, rb, d_.n_embd, st, x);
    CUDA_CHECK(cudaGetLastError()); ++*counter;
}

// One or more passes over `n` mixed rows starting at position n_past: ids[i] >= 0 is a token, ids[i] < 0 is row -1 - ids[i] of emb_host
// (n_emb rows of n_embd floats).  The engine collects consecutive add_tokens / add_embedding calls of a chat turn (reference call sites
// minigpt4.cpp:2365-2382 and :2399-2415 evaluate each piece separately; results are batch invariant) and evaluates them together, so the
// weights stream once per kPrefillMax rows instead of once per piece.
bool LlamaDevice::eval_rows(const int32_t *ids, int n, const float *emb_host, int n_emb, int n_past) {
    if (n <= 0) return true;
    if (n_past + n > d_.n_ctx) { MG4_ERR("context overflow: %d + %d > n_ctx %d", n_past, n, d_.n_ctx); return false; }
    if (n_emb > 512) { MG4_ERR("eval_rows: at most 512 embedding rows per call"); return false; }
    for (int i = 0; i < n; ++i) if (ids[i] >= d_.n_vocab || ids[i] < -n_emb) { MG4_ERR("token id %d out of range", ids[i]); return false; }
    if (n_emb > 0) CUDA_CHECK(cudaMemcpyAsync(embd_in_, emb_host, (size_t)n_emb * d_.n_embd * 4, cudaMemcpyHostToDevice, stream_));
    const int step = pf_ready_ ? kPrefillMax : 8;
    for (int i = 0; i < n; i += step) {
        const int c = std::min(step, n - i);
        CUDA_CHECK(cudaStreamSynchronize(stream_));  // h_state_ (pinned) of the previous pass / decode step has been consumed
        h_state_->n_past = n_past + i; h_state_->n_tok = c;
        for (int j = 0; j < std::min(c, 8); ++j) h_state_->tokens[j] = ids[i + j] >= 0 ? ids[i + j] : 0;
        CUDA_CHECK(cudaMemcpyAsync(state_, h_state_, offsetof(DeviceState, argmax_key), cudaMemcpyHostToDevice, stream_));
        CUDA_CHECK(cudaMemcpyAsync(tok_ids_, ids + i, (size_t)c * 4, cudaMemcpyHostToDevice, stream_));
        embed_rows_kernel<<<c, 256, 0, stream_>>>(tok_type_, (const unsigned char *)tok_raw_, gg_row_bytes(tok_type_, (size_t)d_.n_embd), d_.n_embd, tok_ids_, embd_in_, x_);
        ++launches_;
        record_pass(c, i + c == n);
    }
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    return true;
}
void LlamaDevice::logits_to_host(float *dst) {
    CUDA_CHECK(cudaMemcpyAsync(dst, logits_, (size_t)d_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}
void LlamaDevice::sync_decode() {
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    h_state_busy_ = false;
}
int32_t LlamaDevice::argmax() {
    sync_decode();
    return *h_argmax_;
}
void LlamaDevice::sync() { CUDA_CHECK(cudaStreamSynchronize(stream_)); h_state_busy_ = false; }
void LlamaDevice::hidden_to_host(float *dst, int n) {
    CUDA_CHECK(cudaMemcpyAsync(dst, x_, (size_t)n * d_.n_embd * 4, cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}

// ------------------------------------------------------------------------------------------------
// tensor-core prefill (llama_prefill.cuh)
// ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn tm_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr; cudaDriverEntryPointQueryResult qr;
        CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
        if (!p || qr != cudaDriverEntryPointSuccess) MG4_PANIC("cuTensorMapEncodeTiled is not available from this driver");
        fn = (EncodeTiledFn)p;
    }
    return fn;
}
// bytes [rows][pitch] -> boxes of box_bytes x box_rows
static void make_map_u8(void *tm, const void *ptr, size_t rows, size_t pitch, int box_bytes, int box_rows, bool swizzle128) {
    cuuint64_t dims[2] = {(cuuint64_t)pitch, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)pitch};
    cuuint32_t box[2] = {(cuuint32_t)box_bytes, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = tm_encode_fn()((CUtensorMap *)tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void *)ptr, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) MG4_PANIC("cuTensorMapEncodeTiled failed (%d) for [%zu x %zu] box %d x %d", (int)r, rows, pitch, box_bytes, box_rows);
}
static int pf_slots(int cols) { const int nbl = (cols / 32 + 31) / 32; return 4 * ((nbl + 3) / 4); }

static void pq_build(PQMat &p, const QMat &m) {
    p.rows = m.rows; p.rows_pad = (m.rows + 127) & ~127; p.cols = m.cols; p.nb = m.cols / 32; p.S = pf_slots(m.cols); p.q41 = m.type == GG_Q4_1;
    const size_t pitch = (size_t)32 * p.S * 32;
    dmalloc(&p.q, (size_t)p.rows_pad * pitch); CUDA_CHECK(cudaMemset(p.q, 0, (size_t)p.rows_pad * pitch));
    dmalloc(&p.sc, (size_t)p.rows_pad * 32 * p.S * 4); CUDA_CHECK(cudaMemset(p.sc, 0, (size_t)p.rows_pad * 32 * p.S * 4));
    const size_t n = (size_t)m.rows * p.nb;
    pf::expand_q4_classmajor<<<(unsigned)((n + 255) / 256), 256>>>((const unsigned char *)m.p0, m.row_bytes, m.rows, p.nb, p.q41 ? 1 : 0, p.S, p.q, (__half2 *)p.sc);
    CUDA_CHECK(cudaGetLastError());
    make_map_u8(p.tm, p.q, (size_t)p.rows_pad, pitch, 128, pf::kRows, true);
}

bool LlamaDevice::build_prefill() {
    if (getenv("MINIGPT4_B200_NO_PREFILL_GEMM")) return false;
    if (tp_ && tp_->world > 1) return false;  // (tensor-parallel ranks keep the per-op prefill path for now)
    // (any token-embedding type the loader accepts: prompt rows are gathered by embed_rows_kernel, which decodes every one of them, on both
    // prefill paths - tests/test_mixed_types_gpu.py)
    for (auto &L : layers_) {   // (each matrix stages its own input: mixed Q4_0 / Q4_1 layers are fine)
        if (!L.fused_qkv) return false;
        for (const QMat *m : {&L.qkv, &L.wo, &L.w13, &L.w2}) if (m->type != GG_Q4_0 && m->type != GG_Q4_1) return false;
    }
    const int E = d_.n_embd, FF = d_.n_ff;
    size_t free_b = 0, total_b = 0; CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    const size_t need = (size_t)d_.n_layer * ((size_t)4 * E * E + (size_t)3 * E * (size_t)32 * pf_slots(FF) * 32 / 1) + ((size_t)1 << 30);
    if (need > free_b) { MG4_INFO("prefill operand cache (%.1f GB) does not fit: per-op prefill path", need / 1073741824.0); return false; }
    for (auto &L : layers_) { pq_build(L.pqkv, L.qkv); pq_build(L.pwo, L.wo); pq_build(L.pw13, L.w13); pq_build(L.pw2, L.w2); }
    pf_S_e_ = pf_slots(E); pf_S_ff_ = pf_slots(FF);
    const size_t pitch_e = (size_t)32 * pf_S_e_ * 32, pitch_ff = (size_t)32 * pf_S_ff_ * 32, R = (size_t)kPrefillMax;
    dmalloc(&pf_q8_, R * std::max(pitch_e, pitch_ff)); CUDA_CHECK(cudaMemset(pf_q8_, 0, R * std::max(pitch_e, pitch_ff)));
    dmalloc(&pf_sc_, R * std::max(pitch_e, pitch_ff) / 4); CUDA_CHECK(cudaMemset(pf_sc_, 0, R * std::max(pitch_e, pitch_ff) / 4));
    make_map_u8(pf_tmB_e_, pf_q8_, R, pitch_e, 128, pf::kTok, true);
    make_map_u8(pf_tmS_e_, pf_sc_, R, pitch_e / 4, 32, pf::kTok, false);
    make_map_u8(pf_tmB_ff_, pf_q8_, R, pitch_ff, 128, pf::kTok, true);
    make_map_u8(pf_tmS_ff_, pf_sc_, R, pitch_ff / 4, 32, pf::kTok, false);
    pf_part_bytes_ = (size_t)96 << 20;   // roots of K-split slices: [slice][token][row] {d-tree, m-tree}
    dmalloc(&pf_part_, pf_part_bytes_);
    const size_t smem = 1024 + (size_t)pf::kStages * pf::kStageBytes + pf::kStackBytes + 256;
    CUDA_CHECK(cudaFuncSetAttribute(pf::prefill_gemm_q4<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_CHECK(cudaFuncSetAttribute(pf::prefill_gemm_q4<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CUDA_CHECK(cudaDeviceSynchronize());
    MG4_INFO("tensor-core prefill: int8 class-major operand cache built (%d / %d slots per class)", pf_S_e_, pf_S_ff_);
    return true;
}

void LlamaDevice::pf_stage(const QMat &w, const float *x, int x_stride, const float *nw, int S, const Pass &ps) {
    const int act = act_of(w.type), n = ps.rows;
    const size_t sm = act_bytes(act, w.cols);
    if (act == ACT_Q8_1) pf::stage_rows_classmajor<ACT_Q8_1><<<n, 256, sm, ps.s>>>(x, x_stride, nw, w.cols, S, pf_q8_, (float2 *)pf_sc_);
    else pf::stage_rows_classmajor<ACT_Q8_0><<<n, 256, sm, ps.s>>>(x, x_stride, nw, w.cols, S, pf_q8_, (float2 *)pf_sc_);
    ++*ps.counter;
}
void LlamaDevice::pf_gemm(const PQMat &p, bool ff_wide, const pf::PrefillArgs &epi, const Pass &ps) {
    const size_t smem = 1024 + (size_t)pf::kStages * pf::kStageBytes + pf::kStackBytes + 256;
    const int n = ps.rows;
    const unsigned ty = (unsigned)((n + pf::kTok - 1) / pf::kTok);
    pf::PrefillArgs a = epi;
    a.rows = p.rows; a.n_tok = n; a.nb = p.nb; a.S = p.S; a.wsc = (const __half2 *)p.sc; a.state = ps.state; a.tab_silu = tab_silu_;
    const CUtensorMap *tb = (const CUtensorMap *)(ff_wide ? pf_tmB_ff_ : pf_tmB_e_), *ts = (const CUtensorMap *)(ff_wide ? pf_tmS_ff_ : pf_tmS_e_);
    // K split over subtrees of the class butterfly so that matrices with few 128-row tiles (wo / down: 32) still fill the machine
    const int tiles = p.rows_pad / pf::kRows;
    int nz = 1;
    if (!getenv("MINIGPT4_B200_PREFILL_NO_KSPLIT")) {   // waves of CTAs x work per CTA (+ a little per-CTA overhead), smallest wins
        double best = 1e30;
        for (int c = 1; c <= 8; c *= 2) {
            if ((size_t)c * n * p.rows_pad * sizeof(float2) > pf_part_bytes_ && c > 1) break;
            const int ctas = tiles * (int)ty * c;
            const double cost = (double)((ctas + sm_count_ - 1) / sm_count_) / c + 0.02 * c;
            if (cost < best - 1e-9) { best = cost; nz = c; }
        }
    }
    a.jr_per_z = 32 / nz; a.partial = (float2 *)pf_part_; a.part_tok = n; a.part_rows = p.rows_pad;
    const dim3 grid((unsigned)tiles, ty, (unsigned)nz);
    if (p.q41) pf::prefill_gemm_q4<true><<<grid, pf::kThreads, smem, ps.s>>>(*(const CUtensorMap *)p.tm, *tb, *ts, a);
    else pf::prefill_gemm_q4<false><<<grid, pf::kThreads, smem, ps.s>>>(*(const CUtensorMap *)p.tm, *tb, *ts, a);
    ++*ps.counter;
    if (nz > 1) { const size_t work = (size_t)n * (p.rows / 2); pf::prefill_combine<<<(unsigned)((work + 255) / 256), 256, 0, ps.s>>>(a, nz); ++*ps.counter; }
}

// ------------------------------------------------------------------------------------------------
// persistent megakernel program (llama_mega6.cuh)
// ------------------------------------------------------------------------------------------------
bool LlamaDevice::build_mega() {
    if (getenv("MINIGPT4_B200_NO_MEGAKERNEL")) return false;
    const bool tp = tp_ && tp_->world > 1;
    if (tp && (!tp_->peers_ready() || getenv("MINIGPT4_B200_TP_PER_OP"))) return false;   // the in-kernel all-reduce needs the peer mappings
    const int wt = output_.type;
    if (wt != GG_Q4_0 && wt != GG_Q4_1 && wt != GG_Q5_K) return false;   // homogeneous Q4_0 / Q4_1 / Q5_K files (the reference README's q5_k download has a Q6_K output matrix: per-op path)
    for (auto &L : layers_) if (!L.fused_qkv || L.qkv.type != wt || L.wo.type != wt || L.w13.type != wt || L.w2.type != wt) return false;
    // OP_EMBED decodes the token row with dequant_elem, which knows F32 / F16 / Q4_0 / Q4_1 / Q5_K / Q6_K only (any other type would embed
    // zeros); Q4_K / Q5_0 / Q5_1 / Q8_0 token embeddings take the per-op graph, whose launch_embed decodes them
    if (!(tok_type_ == GG_F32 || tok_type_ == GG_F16 || tok_type_ == GG_Q4_0 || tok_type_ == GG_Q4_1 || tok_type_ == GG_Q5_K || tok_type_ == GG_Q6_K)) return false;
    if (d_.n_embd % 256 || d_.n_ff % 32 || d_.n_embd > 1024 * mk6::kNormItems || d_.n_ff > 4 * mk6::kConsumerThreads * mk6::kPlainItems) return false;
    if (d_.head_dim != 128 || d_.n_head > sm_count_ || 7 * d_.n_layer + 3 > mk6::kMaxOps) return false;
    if (tp && (n_embd_local_ % 32 || n_ff_local_ % 32)) return false;
    int coop = 0, dev = 0; CUDA_CHECK(cudaGetDevice(&dev));
    CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
    if (!coop) return false;
    mega_type_ = wt;
    dmalloc(&mega_barrier_, 64); CUDA_CHECK(cudaMemset(mega_barrier_, 0, 64));
    mega_n_ops_ = (tp ? 7 : 5) * d_.n_layer + 3;
    if (getenv("MINIGPT4_B200_MEGA_TRACE")) { dmalloc(&mega_trace_, (size_t)(mega_n_ops_ + 1) * 32 * sizeof(long long)); CUDA_CHECK(cudaMemset(mega_trace_, 0, (size_t)(mega_n_ops_ + 1) * 32 * sizeof(long long))); }

    // generation 6: self-refilled per-warp streams
    using namespace mk6;
    const int E = d_.n_embd, FF = n_ff_local_;   // (tensor parallel: this rank's feed-forward columns)
    size_t act_b = mega_type_ == GG_Q5_K ? std::max(act_bytes(ACT_Q8_K, FF), act_bytes(ACT_Q8_K, E)) : std::max(act6_bytes(FF), act6_bytes(E));
    act_b = std::max(act_b, (size_t)d_.n_ctx * 6);  // the attention op (which stages no activations) uses the region as its scratch
    act_b = (act_b + 127) & ~(size_t)127;
    if (mega_type_ == GG_Q5_K && (E % 256 || FF % 256 || FF > 256 * kConsumerWarps * kQ8kRounds || E > 256 * kConsumerWarps * 2)) return false;
    const int rb_e = layers_[0].qkv.row_bytes, rb_ff = layers_[0].w2.row_bytes;
    // a slot holds a row pair of an n_embd-wide matrix or ONE row of an n_ff-wide matrix (whose pair then takes both slots of the warp)
    int slot = std::max(2 * rb_e, rb_ff);
    slot = (slot + 15) & ~15;
    cudaDeviceProp prop; CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    const size_t stat = 10240;  // static shared memory of decode_megakernel6 (red, redf, qh, part) + slack
    const long long room = (long long)prop.sharedMemPerBlockOptin - (long long)stat - (long long)act_b - 2 * kConsumerWarps * 8;
    int W = (int)std::min<long long>(kConsumerWarps, room / (2LL * slot));
    if (getenv("MINIGPT4_B200_MEGA_W")) W = std::min(W, atoi(getenv("MINIGPT4_B200_MEGA_W")));
    if (W < 4) return false;
    Params6 *P = new Params6();
    memset(P, 0, sizeof(Params6));
    int n = 0; bool uniform = true;   // every layer's matrices have the same shapes (the CTA's share of a kind is computed once)
    auto add = [&](int kind, int layer, const QMat *m, const float *norm) {
        Op6 &o = P->ops[n++]; o.kind = (unsigned char)kind; o.layer = (unsigned short)layer; o.norm_w = norm;
        if (m) {
            o.cols = m->cols; o.row_bytes = m->row_bytes; o.w = (const unsigned char *)m->p0;
            o.parts = (unsigned char)(2 * m->row_bytes <= slot ? 1 : 2);
            o.n_su = m->rows / 2;
            if ((2 * m->row_bytes / o.parts) % 16) uniform = false;   // every slot-load is a 16-byte aligned, 16-byte multiple bulk copy
            if (P->n_su_kind[kind] && P->n_su_kind[kind] != o.n_su) uniform = false;
            P->n_su_kind[kind] = o.n_su;
        }
    };
    add(OP_EMBED, 0, nullptr, nullptr);
    for (int il = 0; il < d_.n_layer; ++il) {
        Layer &L = layers_[(size_t)il];
        add(OP_QKV, il, &L.qkv, L.attn_norm);
        add(OP_ATTN, il, nullptr, nullptr);
        add(OP_WO, il, &L.wo, nullptr);
        if (tp) add(OP_REDUCE, 0, nullptr, nullptr);   // (`layer` = exchange buffer: 0 after wo, 1 after down)
        add(OP_GATEUP, il, &L.w13, L.ffn_norm);
        add(OP_DOWN, il, &L.w2, nullptr);
        if (tp) add(OP_REDUCE, 1, nullptr, nullptr);
    }
    add(OP_OUTPUT, 0, &output_, final_norm_);
    add(OP_FINAL, 0, nullptr, nullptr);
    if (!uniform) { delete P; return false; }
    P->n_ops = n; P->W = W; P->slot_bytes = slot; P->act_bytes = (int)act_b;
    P->E = E; P->FF = FF; P->n_head = n_head_local_; P->n_ctx = d_.n_ctx; P->n_vocab = d_.n_vocab;
    P->El = n_embd_local_;
    if (tp) { P->tp = tp_->peers; P->tp_seq = tp_->seq_dev; } else { P->tp.world = 1; P->tp.rank = 0; }
    P->flags = getenv("MINIGPT4_B200_MEGA_FLAGS") ? atoi(getenv("MINIGPT4_B200_MEGA_FLAGS")) : 1;
    P->kq_scale = 1.0f / sqrtf((float)d_.n_embd / (float)d_.n_head);
    P->E_pow2 = (E & (E - 1)) == 0; P->inv_E = 1.0 / (double)E;
    P->x = x_; P->q = q_; P->att = att_; P->act = act_; P->logits = logits_; P->kcache = kcache_; P->vcache = vcache_;
    P->rope = rope_; P->tab_exp = tab_exp_; P->tab_silu = tab_silu_;
    P->tok = (const unsigned char *)tok_raw_; P->tok_type = tok_type_; P->tok_row_bytes = gg_row_bytes(tok_type_, (size_t)E);
    P->state = state_; P->barrier = mega_barrier_; P->trace = mega_trace_;
    mega6_params_ = P;
    mega6_nbl_ = (getenv("MINIGPT4_B200_MEGA_NOREG") || mega_type_ == GG_Q5_K) ? 0 : E == 4096 ? 4 : E == 5120 ? 5 : 0;
    mega_smem_ = (size_t)2 * W * slot + act_b + (size_t)2 * W * 8;
    MG4_INFO("decode megakernel (generation 6): %d ops/token, %d stream warps x 2 slots x %d B, act %zu B, %zu B dynamic shared per CTA, register-resident blocks per lane %d, grid %d",
             n, W, slot, act_b, mega_smem_, mega6_nbl_, sm_count_);
    const void *fn = mega_fn();
    CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mega_smem_));
    int occ = 0;
    CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, mk6::kThreads, mega_smem_));
    if (occ < 1) { MG4_ERR("megakernel does not fit on an SM (smem %zu)", mega_smem_); return false; }
    return true;
}

const void *LlamaDevice::mega_fn() const {
    const bool t = mega_trace_ != nullptr, q41 = mega_type_ == GG_Q4_1;
    using namespace mk6;
    if (mega_type_ == GG_Q5_K) return t ? (const void *)decode_megakernel6<GG_Q5_K, 0, true> : (const void *)decode_megakernel6<GG_Q5_K, 0, false>;
#define MG4_M6(NBL) (q41 ? (t ? (const void *)decode_megakernel6<GG_Q4_1, NBL, true> : (const void *)decode_megakernel6<GG_Q4_1, NBL, false>) \
                         : (t ? (const void *)decode_megakernel6<GG_Q4_0, NBL, true> : (const void *)decode_megakernel6<GG_Q4_0, NBL, false>))
    return mega6_nbl_ == 4 ? MG4_M6(4) : mega6_nbl_ == 5 ? MG4_M6(5) : MG4_M6(0);
#undef MG4_M6
}
void LlamaDevice::launch_mega() {
    CUDA_CHECK(cudaMemsetAsync(mega_barrier_, 0, 4, stream_));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)sm_count_); cfg.blockDim = dim3(mk6::kThreads); cfg.dynamicSmemBytes = mega_smem_; cfg.stream = stream_;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    void *args[1] = {mega6_params_};
    CUDA_CHECK(cudaLaunchKernelExC(&cfg, mega_fn(), args));
    ++launches_;
    CUDA_CHECK(cudaMemcpyAsync(h_argmax_, &state_->argmax_id, 4, cudaMemcpyDeviceToHost, stream_));
}

// the decode step as a CUDA graph: the megakernel, or embed(tokens[0]) -> layers -> logits/arg-max -> finalize (n_past++, tokens[0] =
// arg-max).  Positions and the token come from *state_, so the same graph serves every step.
void LlamaDevice::build_graph() {
    cudaGraph_t g = nullptr;
    const unsigned long long before = launches_;
    mega_ = build_mega();
    CUDA_CHECK(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
    if (mega_) launch_mega();
    else { launch_embed(1, state_, x_, stream_, &launches_); record_pass(1, true); }
    CUDA_CHECK(cudaStreamEndCapture(stream_, &g));
    CUDA_CHECK(cudaGraphInstantiate(&graph_, g, 0));
    CUDA_CHECK(cudaGraphDestroy(g));
    graph_kernels_ = (int)(launches_ - before);
    launches_ = before;
}
bool LlamaDevice::decode_step(int32_t id, int n_past) {
    if (n_past + 1 > d_.n_ctx) { MG4_ERR("context overflow at %d", n_past); return false; }
    if (id >= 0) {
        if (h_state_busy_) CUDA_CHECK(cudaStreamSynchronize(stream_));  // the previous step's copy out of the pinned state may not have run yet
        h_state_->n_past = n_past; h_state_->n_tok = 1; h_state_->tokens[0] = id;
        CUDA_CHECK(cudaMemcpyAsync(state_, h_state_, offsetof(DeviceState, argmax_key), cudaMemcpyHostToDevice, stream_));
        h_state_busy_ = true;
    }
    CUDA_CHECK(cudaGraphLaunch(graph_, stream_));
    launches_ += (unsigned long long)graph_kernels_;
    return true;
}
float LlamaDevice::decode_chain(int steps, int n_past, int32_t *ids_out) {
    if (n_past + steps > d_.n_ctx) { MG4_ERR("context overflow"); return -1.f; }
    // the chain starts from the device state left by the previous eval: tokens[0] = arg-max, n_past up to date
    int32_t *ids_dev = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&ids_dev, (size_t)steps * 4));
    CUDA_CHECK(cudaEventRecord(ev0_, stream_));
    for (int i = 0; i < steps; ++i) {
        CUDA_CHECK(cudaMemcpyAsync(ids_dev + i, &state_->tokens[0], 4, cudaMemcpyDeviceToDevice, stream_));  // the id being fed
        CUDA_CHECK(cudaGraphLaunch(graph_, stream_));
    }
    CUDA_CHECK(cudaEventRecord(ev1_, stream_));
    sync_decode();
    launches_ += (unsigned long long)graph_kernels_ * steps;
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, ev0_, ev1_));
    if (ids_out) CUDA_CHECK(cudaMemcpy(ids_out, ids_dev, (size_t)steps * 4, cudaMemcpyDeviceToHost));
    cudaFree(ids_dev);
    return ms;
}

// ------------------------------------------------------------------------------------------------
// the group workspace of the batched passes (llama_sessions.cuh), built by the group's first decode_batch or batched flush: kPrefillMax
// rows of activations, a row table for the prompt pass and a context table for the decode step and the contexts that end in a prompt
// pass.  Both users run synchronously on the group stream, so they share it; the batch graphs capture its pointers.
// ------------------------------------------------------------------------------------------------
void LlamaDevice::build_group_workspace() {
    LlamaGroup &G = *group_;
    const int E = d_.n_embd, El = n_embd_local_, FF = d_.n_ff, FFl = n_ff_local_;
    const size_t R = (size_t)kPrefillMax, b0 = t_dev_bytes;
    CUDA_CHECK(cudaStreamCreateWithFlags(&G.stream, cudaStreamNonBlocking));
    dmalloc(&G.x, R * E * 4);
    dmalloc(&G.q, R * El * 4);
    dmalloc(&G.att, R * El * 4);
    dmalloc(&G.act, R * std::max(FFl, 3 * El) * 4);
    dmalloc(&G.last, (size_t)8 * E * 4);
    dmalloc(&G.qact, (size_t)8 * ((size_t)std::max(E, FF) * 2 + 4096));
    dmalloc(&G.state, sizeof(DeviceState)); CUDA_CHECK(cudaMemset(G.state, 0, sizeof(DeviceState)));
    dmalloc(&G.tok, kMaxBatch * sizeof(int));
    dmalloc(&G.rows, R * sizeof(SessionSlot));
    dmalloc(&G.slots, kMaxBatch * sizeof(SessionSlot));
    dmalloc(&G.ids, kMaxBatch * sizeof(int));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_rows, R * sizeof(SessionSlot), cudaHostAllocDefault));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_slots, kMaxBatch * sizeof(SessionSlot), cudaHostAllocDefault));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_ids, kMaxBatch * sizeof(int), cudaHostAllocDefault));
    CUDA_CHECK(cudaDeviceSynchronize());
    G.batch_bytes += t_dev_bytes - b0;
}

// ------------------------------------------------------------------------------------------------
// batched decode step over B contexts of one group: prepare (tokens) -> embed B rows -> layers (QKV and attention per column through the
// context table; wo / gate-up / down through matvec_kernel at ntok = B) -> logits of every column into its own context -> finalize every
// context's DeviceState -> the B ids to pinned memory.  Captured once per B on the group stream.
// More than 8 columns: the tokens go through the group's id list (DeviceState holds 8), the layers run in 8-column matvec chunks or, from
// kWideGemmMin columns on a pf_ready_ model, as the tensor-core pass of the batched prompt pass (one row per column), and the logits in
// 8-column chunks.  Every column still gets the bits of its own decode step.
// ------------------------------------------------------------------------------------------------
void LlamaDevice::build_batch_graph(int B) {
    LlamaGroup &G = *group_;
    cudaStream_t s = G.stream;
    unsigned long long n = 0;
    cudaGraph_t g = nullptr;
    const int E = d_.n_embd, block = (B + 31) / 32 * 32;   // (prepare / finalize: a thread per column)
    CUDA_CHECK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    if (B <= 8) {
        prepare_sessions_kernel<<<1, 32, 0, s>>>(G.slots, B, G.state); ++n;
        launch_embed(B, G.state, G.x, s, &n);
    } else {
        prepare_wide_kernel<<<1, block, 0, s>>>(G.slots, B, G.tok); ++n;
        embed_rows_kernel<<<B, 256, 0, s>>>(tok_type_, (const unsigned char *)tok_raw_, gg_row_bytes(tok_type_, (size_t)E), E, G.tok, embd_in_, G.x); ++n;
    }
    record_layers(Pass{B, G.x, G.q, G.att, G.act, G.qact, G.state, G.slots, pf_ready_ && B >= kWideGemmMin, s, &n});
    for (int t0 = 0; t0 < B; t0 += 8) {
        MatvecArgs o = mv_args(output_, std::min(8, B - t0), G.state, G.qact, tab_silu_);
        o.x = G.x + (size_t)t0 * E; o.x_stride = E; o.norm_w = final_norm_; o.epi = EPI_LOGITS; o.n_valid = d_.n_vocab;
        launch_matvec(o, sm_count_, s, &n, G.slots + t0, 0);
    }
    finalize_sessions_kernel<<<1, block, 0, s>>>(G.slots, B, G.ids); ++n;
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpyAsync(G.h_ids, G.ids, (size_t)B * 4, cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaStreamEndCapture(s, &g));
    CUDA_CHECK(cudaGraphInstantiate(&G.graph[B], g, 0));
    CUDA_CHECK(cudaGraphDestroy(g));
    G.graph_kernels[B] = (int)n;
}

cudaStream_t LlamaDevice::open_batch(LlamaDevice *const *c, int n, const int32_t *ids, const int *n_past) {
    LlamaDevice &L0 = *c[0];
    LlamaGroup &G = *L0.group_;
    // a context's own decode step may still be running on its stream (decode_step returns before it finishes): it has to be done
    // before the group stream reads and writes that context's cache, logits and state
    for (int i = 0; i < n; ++i) c[i]->sync();
    if (!G.x) L0.build_group_workspace();
    if (!G.graph[n]) L0.build_batch_graph(n);
    for (int i = 0; i < n; ++i) G.h_slots[i] = SessionSlot{n_past[i], ids ? ids[i] : -1, c[i]->kcache_, c[i]->vcache_, c[i]->logits_, c[i]->state_};
    CUDA_CHECK(cudaMemcpyAsync(G.slots, G.h_slots, (size_t)n * sizeof(SessionSlot), cudaMemcpyHostToDevice, G.stream));
    return G.stream;
}

void LlamaDevice::decode_batch(LlamaDevice *const *c, int n, const int32_t *ids, const int *n_past, int32_t *ids_out) {
    LlamaDevice &L0 = *c[0];
    LlamaGroup &G = *L0.group_;
    open_batch(c, n, ids, n_past);
    CUDA_CHECK(cudaGraphLaunch(G.graph[n], G.stream));
    CUDA_CHECK(cudaStreamSynchronize(G.stream));   // (h_slots / h_ids are reused by the next step)
    L0.launches_ += (unsigned long long)G.graph_kernels[n];
    for (int i = 0; i < n; ++i) { ids_out[i] = G.h_ids[i]; *c[i]->h_argmax_ = G.h_ids[i]; }
}

// ------------------------------------------------------------------------------------------------
// batched prompt pass over the queued rows of several contexts of one group.  Each pass takes the next <= kPrefillMax rows of the
// contexts in order; row t carries its own position and its context's caches in the row table, and record_layers runs the pass with it.
// Contexts whose last row is in the pass get their logits, arg-max and DeviceState through the context table, as the batched decode
// step does.  Every row is quantised and reduced on its own, so each context gets the bits of its own eval_rows.
// A scoring pass (score_rows) points each row's logits at its row of the group's scratch instead: after the layers every row's logits
// are computed in 8-row chunks straight from the pass's rows, the entries whose logits are in this pass are scored, and the results and
// requested logits rows go to the host.  The context tail runs only with score->keep.
// ------------------------------------------------------------------------------------------------
struct ScoreCall {
    bool keep;
    float *const *logprob;    // [n] entries of each context
    int32_t *const *rank;     // [n] or null
    float *const *logits;     // [n] rows of n_vocab of each context, or null
};

void LlamaDevice::eval_rows_batch(LlamaDevice *const *c, int n, const int32_t *const *ids, const int *n_rows, const float *const *emb, const int *n_past,
                                  const ScoreCall *score) {
    LlamaDevice &L0 = *c[0];
    LlamaGroup &G = *L0.group_;
    for (int i = 0; i < n; ++i) c[i]->sync();   // (as decode_batch: a context's own work must be done before the group stream uses its memory)
    if (!G.x) L0.build_group_workspace();
    if (score && !G.score_logits) L0.build_score_scratch();
    const int E = L0.d_.n_embd, S = kPrefillMax;
    const size_t V = (size_t)L0.d_.n_vocab;
    cudaStream_t s = G.stream;
    std::vector<int32_t> pid((size_t)S);
    std::vector<int> ent_ctx, ent_j;   // scoring: each entry's context and index, in the order of the pass's entry table
    int ci = 0, cj = 0;   // next row: row cj of context ci
    while (ci < n) {
        // ---- the pass: rows, their slots and ids; embedding rows of each context are a contiguous run of its emb[] (queued in order)
        int rows = 0, n_emb = 0, nf = 0, nr = 0;
        int last[kMaxBatch], fin_ctx[kMaxBatch], fin_first[kMaxBatch];
        int run_ctx[kMaxBatch], run_j[kMaxBatch], run_row[kMaxBatch], run_n[kMaxBatch];   // scoring: each context's rows in this pass
        ent_ctx.clear(); ent_j.clear();
        for (; ci < n && rows < S; ++ci, cj = 0) {
            const int take = std::min(n_rows[ci] - cj, S - rows);
            LlamaDevice &X = *c[ci];
            int k0 = -1, k1 = -1;
            for (int j = 0; j < take; ++j) {
                const int id = ids[ci][cj + j], r = rows + j;
                if (!score) G.h_rows[r] = SessionSlot{n_past[ci] + cj + j, 0, X.kcache_, X.vcache_, X.logits_, X.state_};
                else {
                    G.h_rows[r] = SessionSlot{n_past[ci] + cj + j, 0, X.kcache_, X.vcache_, G.score_logits + (size_t)r * V, G.score_state};
                    const int jj = cj + j;
                    if (jj == 0 && n_past[ci] > 0) {   // entry 0: the logits the context holds now (read before any tail of this call)
                        G.h_score_rows[ent_ctx.size()] = k::ScoreRow{X.logits_, id, 0};
                        ent_ctx.push_back(ci); ent_j.push_back(0);
                    } else if (jj == 0) {
                        score->logprob[ci][0] = NAN;
                        if (score->rank) score->rank[ci][0] = -1;
                    }
                    if (jj + 1 < n_rows[ci]) {         // entry jj + 1: this row's logits
                        G.h_score_rows[ent_ctx.size()] = k::ScoreRow{G.score_logits + (size_t)r * V, ids[ci][jj + 1], 0};
                        ent_ctx.push_back(ci); ent_j.push_back(jj + 1);
                    }
                }
                if (id >= 0) pid[(size_t)r] = id;
                else {
                    const int k = -1 - id;
                    if (k0 < 0) k0 = k;
                    k1 = k;
                    pid[(size_t)r] = -1 - (n_emb + k - k0);
                }
            }
            if (k0 >= 0) {
                CUDA_CHECK(cudaMemcpyAsync(L0.embd_in_ + (size_t)n_emb * E, emb[ci] + (size_t)k0 * E, (size_t)(k1 - k0 + 1) * E * 4, cudaMemcpyHostToDevice, s));
                n_emb += k1 - k0 + 1;
            }
            run_ctx[nr] = ci; run_j[nr] = cj; run_row[nr] = rows; run_n[nr] = take; ++nr;
            rows += take; cj += take;
            if (cj < n_rows[ci]) break;   // the context continues in the next pass
            G.h_slots[nf] = SessionSlot{n_past[ci] + n_rows[ci] - 1, 0, X.kcache_, X.vcache_, X.logits_, X.state_};
            last[nf] = rows - 1; fin_ctx[nf] = ci; fin_first[nf] = rows - take;
            ++nf;
        }
        const bool tail = nf && (!score || score->keep);
        CUDA_CHECK(cudaMemcpyAsync(G.rows, G.h_rows, (size_t)rows * sizeof(SessionSlot), cudaMemcpyHostToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(L0.tok_ids_, pid.data(), (size_t)rows * 4, cudaMemcpyHostToDevice, s));
        if (tail) CUDA_CHECK(cudaMemcpyAsync(G.slots, G.h_slots, (size_t)nf * sizeof(SessionSlot), cudaMemcpyHostToDevice, s));
        embed_rows_kernel<<<rows, 256, 0, s>>>(L0.tok_type_, (const unsigned char *)L0.tok_raw_, gg_row_bytes(L0.tok_type_, (size_t)E), E, L0.tok_ids_, L0.embd_in_, G.x);
        ++L0.launches_;
        L0.record_layers(Pass{rows, G.x, G.q, G.att, G.act, G.qact, G.state, G.rows, L0.pf_ready_ && rows >= 2, s, &L0.launches_});

        // ---- scoring: every row's logits into the scratch, the entries of this pass, results and logits rows to the host
        const int ne = (int)ent_ctx.size();
        if (score) {
            for (int t0 = 0; t0 < rows; t0 += 8) {
                MatvecArgs o = mv_args(L0.output_, std::min(8, rows - t0), G.state, G.qact, L0.tab_silu_);
                o.x = G.x + (size_t)t0 * E; o.x_stride = E; o.norm_w = L0.final_norm_; o.epi = EPI_LOGITS; o.n_valid = (int)V;
                launch_matvec(o, L0.sm_count_, s, &L0.launches_, G.rows + t0, 0);
            }
            if (ne) {
                CUDA_CHECK(cudaMemcpyAsync(G.score_rows, G.h_score_rows, (size_t)ne * sizeof(k::ScoreRow), cudaMemcpyHostToDevice, s));
                score_rows_kernel<<<ne, 256, 0, s>>>(G.score_rows, (int)V, G.score_out);
                CUDA_CHECK(cudaGetLastError()); ++L0.launches_;
                CUDA_CHECK(cudaMemcpyAsync(G.h_score_out, G.score_out, (size_t)ne * sizeof(k::ScoreOut), cudaMemcpyDeviceToHost, s));
            }
            if (score->logits)
                for (int u = 0; u < nr; ++u)
                    CUDA_CHECK(cudaMemcpyAsync(score->logits[run_ctx[u]] + (size_t)run_j[u] * V, G.score_logits + (size_t)run_row[u] * V,
                                               (size_t)run_n[u] * V * 4, cudaMemcpyDeviceToHost, s));
        }

        // ---- contexts that end in this pass, 8 at a time: logits + arg-max of their last row, DeviceState; then hidden rows, pinned arg-max
        if (tail) {
            for (int f0 = 0; f0 < nf; f0 += 8) {
                const int m = std::min(8, nf - f0);
                RowList lr{};
                for (int f = 0; f < m; ++f) lr.r[f] = last[f0 + f];
                gather_rows_kernel<<<m, 256, 0, s>>>(G.x, lr, E, G.last);
                prepare_sessions_kernel<<<1, 32, 0, s>>>(G.slots + f0, m, G.state);
                MatvecArgs o = mv_args(L0.output_, m, G.state, G.qact, L0.tab_silu_);
                o.x = G.last; o.x_stride = E; o.norm_w = L0.final_norm_; o.epi = EPI_LOGITS; o.n_valid = L0.d_.n_vocab;
                launch_matvec(o, L0.sm_count_, s, &L0.launches_, G.slots + f0, 0);
                finalize_sessions_kernel<<<1, 32, 0, s>>>(G.slots + f0, m, G.ids + f0);
                CUDA_CHECK(cudaGetLastError()); L0.launches_ += 3;
            }
            CUDA_CHECK(cudaMemcpyAsync(G.h_ids, G.ids, (size_t)nf * 4, cudaMemcpyDeviceToHost, s));
            for (int f = 0; f < nf; ++f) {
                const int k = last[f] + 1 - fin_first[f];
                CUDA_CHECK(cudaMemcpyAsync(c[fin_ctx[f]]->x_, G.x + (size_t)fin_first[f] * E, (size_t)k * E * 4, cudaMemcpyDeviceToDevice, s));
            }
        }
        CUDA_CHECK(cudaStreamSynchronize(s));   // (the pinned tables and the shared workspace are reused by the next pass)
        if (tail) for (int f = 0; f < nf; ++f) *c[fin_ctx[f]]->h_argmax_ = G.h_ids[f];
        for (int e = 0; e < ne; ++e) {
            score->logprob[ent_ctx[(size_t)e]][ent_j[(size_t)e]] = G.h_score_out[e].logprob;
            if (score->rank) score->rank[ent_ctx[(size_t)e]][ent_j[(size_t)e]] = G.h_score_out[e].rank;
        }
    }
}

void LlamaDevice::build_score_scratch() {
    LlamaGroup &G = *group_;
    const size_t b0 = t_dev_bytes, R = (size_t)kPrefillMax, NE = R + kMaxBatch;
    dmalloc(&G.score_logits, R * (size_t)d_.n_vocab * 4);
    dmalloc(&G.score_state, sizeof(DeviceState)); CUDA_CHECK(cudaMemset(G.score_state, 0, sizeof(DeviceState)));
    dmalloc(&G.score_rows, NE * sizeof(k::ScoreRow));
    dmalloc(&G.score_out, NE * sizeof(k::ScoreOut));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_score_rows, NE * sizeof(k::ScoreRow), cudaHostAllocDefault));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_score_out, NE * sizeof(k::ScoreOut), cudaHostAllocDefault));
    CUDA_CHECK(cudaDeviceSynchronize());
    G.batch_bytes += t_dev_bytes - b0;
}

void LlamaDevice::score_rows(LlamaDevice *const *c, int n, const int32_t *const *ids, const int *n_ids, const int *n_past, bool keep,
                             float *const *logprob, int32_t *const *rank, float *const *logits) {
    const ScoreCall sc{keep, logprob, rank, logits};
    eval_rows_batch(c, n, ids, n_ids, nullptr, n_past, &sc);
}

// ------------------------------------------------------------------------------------------------
// conversation copies (llama_state.cuh) and save / restore through host memory
// ------------------------------------------------------------------------------------------------
unsigned long long LlamaDevice::fingerprint() const { return group_->fingerprint; }

float LlamaDevice::copy_state(LlamaDevice &src, LlamaDevice *const *dst, int n, int n_past) {
    // a context's own step may still be running (minigpt4_end_chat returns before it finishes): every context involved has to be idle
    src.sync();
    for (int i = 0; i < n; ++i) dst[i]->sync();
    const LlamaDims &d = src.d_;
    const long long row = (long long)src.n_embd_local_ * 2 / 16;   // 16-byte chunks of one cache row
    CopyStateArgs a{};
    a.k = (const uint4 *)src.kcache_; a.v = (const uint4 *)src.vcache_; a.logits = src.logits_; a.state = src.state_;
    for (int i = 0; i < n; ++i) { a.dk[i] = (uint4 *)dst[i]->kcache_; a.dv[i] = (uint4 *)dst[i]->vcache_; a.dlogits[i] = dst[i]->logits_; a.dstate[i] = dst[i]->state_; }
    a.plane = (long long)d.n_ctx * row; a.run = (long long)n_past * row; a.n = n; a.n_layer = d.n_layer; a.n_vocab = d.n_vocab;
    // about two waves over the 2 n_layer planes, no more blocks than a plane has chunks for (the logits row needs one block per
    // kCopyThreads logits, which the KV rows outnumber from a few rows on)
    static int per_sm = 0;
    if (!per_sm) CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, copy_state_kernel, kCopyThreads, 0));
    const long long per_plane = std::max(1LL, 2LL * per_sm * src.sm_count_ / (2 * d.n_layer));
    const long long need = std::max((a.run + kCopyThreads - 1) / kCopyThreads, (long long)(d.n_vocab + kCopyThreads - 1) / kCopyThreads);
    const dim3 grid((unsigned)std::max(1LL, std::min(per_plane, need)), (unsigned)(2 * d.n_layer + 1));
    CUDA_CHECK(cudaEventRecord(src.ev0_, src.stream_));
    copy_state_kernel<<<grid, kCopyThreads, 0, src.stream_>>>(a);
    CUDA_CHECK(cudaGetLastError()); ++src.launches_;
    CUDA_CHECK(cudaEventRecord(src.ev1_, src.stream_));
    CUDA_CHECK(cudaStreamSynchronize(src.stream_));
    for (int i = 0; i < n; ++i) *dst[i]->h_argmax_ = *src.h_argmax_;
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, src.ev0_, src.ev1_));
    return ms;
}

void LlamaDevice::state_to_host(int n_past, DeviceState *st, float *logits, void *kv) {
    sync();
    const size_t run = (size_t)n_past * n_embd_local_ * 2, plane = (size_t)d_.n_ctx * n_embd_local_;
    CUDA_CHECK(cudaMemcpyAsync(st, state_, sizeof(DeviceState), cudaMemcpyDeviceToHost, stream_));
    CUDA_CHECK(cudaMemcpyAsync(logits, logits_, (size_t)d_.n_vocab * 4, cudaMemcpyDeviceToHost, stream_));
    unsigned char *out = (unsigned char *)kv;
    if (run)
        for (int p = 0; p < 2 * d_.n_layer; ++p) {
            const __half *c = (p < d_.n_layer ? kcache_ : vcache_) + (size_t)(p % d_.n_layer) * plane;
            CUDA_CHECK(cudaMemcpyAsync(out + (size_t)p * run, c, run, cudaMemcpyDeviceToHost, stream_));
        }
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}

void LlamaDevice::state_from_host(int n_past, const DeviceState &st, const float *logits, const void *kv) {
    sync();
    const size_t run = (size_t)n_past * n_embd_local_ * 2, plane = (size_t)d_.n_ctx * n_embd_local_;
    *h_state_ = st;
    CUDA_CHECK(cudaMemcpyAsync(state_, h_state_, sizeof(DeviceState), cudaMemcpyHostToDevice, stream_));
    CUDA_CHECK(cudaMemcpyAsync(logits_, logits, (size_t)d_.n_vocab * 4, cudaMemcpyHostToDevice, stream_));
    const unsigned char *in = (const unsigned char *)kv;
    if (run)
        for (int p = 0; p < 2 * d_.n_layer; ++p) {
            __half *c = (p < d_.n_layer ? kcache_ : vcache_) + (size_t)(p % d_.n_layer) * plane;
            CUDA_CHECK(cudaMemcpyAsync(c, in + (size_t)p * run, run, cudaMemcpyHostToDevice, stream_));
        }
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    *h_argmax_ = st.argmax_id;
}

// measurement seam: average CUDA-event duration (us) of one all-reduce of a [1, n_embd] partial on the tensor-parallel path in use
// (one-shot peer kernel, or ncclAllReduce + add); every rank must call it with the same reps (even)
bool LlamaDevice::tp_peer_path() const { return tp_ && tp_->world > 1 && tp_->peers_ready(); }
float LlamaDevice::time_allreduce(int reps) {
    if (!tp_ || tp_->world <= 1) return 0.f;
    reps = std::max(2, reps & ~1);
    const int E = d_.n_embd;
    auto one = [&]() {
        if (tp_->peers_ready()) { CUDA_CHECK(cudaMemsetAsync(tp_->partial_out(), 0, (size_t)E * 4, stream_)); tp_->all_reduce_resid(partial_, partial_, (size_t)E, stream_); }
        else { tp_->all_reduce_sum(partial_, (size_t)E, stream_); add_kernel<<<(E + 255) / 256, 256, 0, stream_>>>(partial_, partial_, E); }
    };
    for (int i = 0; i < 4; ++i) one();
    CUDA_CHECK(cudaEventRecord(ev0_, stream_));
    for (int i = 0; i < reps; ++i) one();
    CUDA_CHECK(cudaEventRecord(ev1_, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, ev0_, ev1_));
    return ms * 1e3f / (float)reps;
}
int LlamaDevice::mega_trace(long long *out, int max_values) {
    if (!mega_trace_) return 0;
    const int n = std::min(max_values, mega_n_ops_ * 32);
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    CUDA_CHECK(cudaMemcpy(out, mega_trace_, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost));
    return n;
}
float LlamaDevice::time_matvec(int kind, int reps, double *bytes_per_launch) {
    const int E = d_.n_embd, El = n_embd_local_, FFl = n_ff_local_, C = d_.n_ctx;
    void *flush = nullptr; const size_t flush_bytes = 256u << 20;
    if (kind == 4) CUDA_CHECK(cudaMalloc(&flush, flush_bytes));
    h_state_->n_past = 0; h_state_->n_tok = 1; h_state_->tokens[0] = 1;
    CUDA_CHECK(cudaMemcpyAsync(state_, h_state_, offsetof(DeviceState, argmax_key), cudaMemcpyHostToDevice, stream_));
    double total_ms = 0.0, bytes = 0.0; long launches = 0;
    auto one = [&](int il) {
        Layer &L = layers_[(size_t)(kind == 4 ? 0 : il)];
        MatvecArgs a{};
        a.ntok = 1; a.state = state_; a.tab_silu = tab_silu_; a.staged = qact_;
        switch (kind) {
            case 0: a.w = L.fused_qkv ? L.qkv : L.wq; a.x = x_; a.x_stride = E; a.norm_w = L.attn_norm; a.epi = EPI_QKV; a.q_out = q_;
                    a.kcache = kcache_ + (size_t)il * C * El; a.vcache = vcache_ + (size_t)il * C * El; a.rope = rope_; a.e_local = El; a.half_dim = 64; a.part = L.fused_qkv ? -1 : 0; break;
            case 1: a.w = L.wo; a.x = att_; a.x_stride = El; a.epi = EPI_PLAIN; a.out = partial_; a.out_stride = E; break;
            case 2: a.w = L.w13; a.x = x_; a.x_stride = E; a.norm_w = L.ffn_norm; a.epi = EPI_SWIGLU; a.out = act_; a.out_stride = FFl; break;
            case 3: a.w = L.w2; a.x = act_; a.x_stride = FFl; a.epi = EPI_PLAIN; a.out = partial_; a.out_stride = E; break;
            default: a.w = output_; a.x = x_; a.x_stride = E; a.norm_w = final_norm_; a.epi = EPI_LOGITS; a.out = logits_; a.n_valid = d_.n_vocab; break;
        }
        if (kind != 4) a.n_valid = a.w.rows;
        bytes = (double)a.w.bytes;
        launch_matvec(a, sm_count_, stream_, &launches_);
    };
    for (int il = 0; il < d_.n_layer; ++il) one(il);  // warm-up pass (instruction cache, smem attributes)
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    for (int r = 0; r < reps; ++r) {
        if (kind == 4) {
            for (int i = 0; i < 8; ++i) {
                CUDA_CHECK(cudaMemsetAsync(flush, i, flush_bytes, stream_));  // evict the 50 MB L2
                CUDA_CHECK(cudaEventRecord(ev0_, stream_)); one(0); CUDA_CHECK(cudaEventRecord(ev1_, stream_));
                CUDA_CHECK(cudaStreamSynchronize(stream_));
                float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, ev0_, ev1_)); total_ms += ms; ++launches;
            }
        } else {
            CUDA_CHECK(cudaEventRecord(ev0_, stream_));
            for (int il = 0; il < d_.n_layer; ++il) one(il);
            CUDA_CHECK(cudaEventRecord(ev1_, stream_));
            CUDA_CHECK(cudaStreamSynchronize(stream_));
            float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, ev0_, ev1_)); total_ms += ms; launches += d_.n_layer;
        }
    }
    if (flush) cudaFree(flush);
    CUDA_CHECK(cudaMemsetAsync(&state_->argmax_key, 0, 8, stream_));
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    if (bytes_per_launch) *bytes_per_launch = bytes;
    return (float)(total_ms / (double)launches);
}

// ------------------------------------------------------------------------------------------------
void LlamaDevice::test_matvec(int gg, int rows, int cols, const void *w_host, const float *x_host, int n, float *y_host) {
    if (!type_supported(gg)) MG4_PANIC("test_matvec: unsupported type %d", gg);
    int dev = 0; CUDA_CHECK(cudaGetDevice(&dev));
    cudaDeviceProp prop; CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
    if (!g_max_dyn_smem) g_max_dyn_smem = std::min<size_t>(prop.sharedMemPerBlockOptin, 220 * 1024) - 1024;
    HostTensor t; t.gg = gg; t.n_dims = 2; t.ne[0] = cols; t.ne[1] = rows; t.data = (const uint8_t *)w_host; t.nbytes = (size_t)rows * gg_row_bytes(gg, (size_t)cols);
    QMat m; Stager st;
    qmat_alloc(m, gg, rows, cols);
    repack_into(m, t, st, 0, rows, 0, cols, 1, 0, 0);
    float *x, *y; DeviceState *stt; unsigned char *stg;
    CUDA_CHECK(cudaMalloc((void **)&stg, (size_t)8 * ((size_t)cols * 2 + 4096)));
    CUDA_CHECK(cudaMalloc((void **)&x, (size_t)n * cols * 4)); CUDA_CHECK(cudaMalloc((void **)&y, (size_t)n * m.rows * 4));
    CUDA_CHECK(cudaMalloc((void **)&stt, sizeof(DeviceState))); CUDA_CHECK(cudaMemset(stt, 0, sizeof(DeviceState)));
    CUDA_CHECK(cudaMemcpy(x, x_host, (size_t)n * cols * 4, cudaMemcpyHostToDevice));
    for (int i = 0; i < n; i += 8) {
        const int c = std::min(8, n - i);
        MatvecArgs a{};
        a.w = m; a.x = x + (size_t)i * cols; a.x_stride = cols; a.ntok = c; a.epi = EPI_PLAIN; a.out = y + (size_t)i * m.rows; a.out_stride = m.rows; a.n_valid = rows; a.state = stt; a.staged = stg;
        launch_matvec(a, prop.multiProcessorCount, 0, nullptr);
    }
    CUDA_CHECK(cudaDeviceSynchronize());
    std::vector<float> tmp((size_t)n * m.rows);
    CUDA_CHECK(cudaMemcpy(tmp.data(), y, tmp.size() * 4, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) memcpy(y_host + (size_t)i * rows, tmp.data() + (size_t)i * m.rows, (size_t)rows * 4);
    cudaFree(x); cudaFree(y); cudaFree(stt); cudaFree(stg); qmat_free(m);
}

// kernel-level test hook of the decode / prompt attention: attn_kernel (path 0, row t at pos[0] + t, the single-context graphs) or
// attn_sessions_kernel (path 1, row t at pos[t] through a slot table, the batched passes) over caller-supplied F16 caches
bool LlamaDevice::test_attention(const float *q_host, const uint16_t *k_host, const uint16_t *v_host, int n_head, int n_ctx, int rows, const int *pos,
                                 int path, float *out_host) {
    if (n_head < 1 || n_head > 128 || n_ctx < 8 || n_ctx > 32768 || rows < 1 || rows > 65535 || (path != 0 && path != 1)) return false;
    for (int t = 0; t < rows; ++t) if (pos[t] < 0 || pos[t] >= n_ctx) return false;
    if (path == 0 && pos[0] + rows > n_ctx) return false;
    const int E = n_head * 128;
    const float kq_scale = 1.0f / sqrtf((float)E / (float)n_head);   // record_layers' expression
    const size_t kv = (size_t)n_ctx * E;
    std::vector<unsigned short> te(65536), ts(65536);
    fp16_tables(te.data(), ts.data());
    float *q, *out; __half *kc, *vc, *tab_exp; DeviceState *st; SessionSlot *slots;
    CUDA_CHECK(cudaMalloc((void **)&q, (size_t)rows * E * 4)); CUDA_CHECK(cudaMalloc((void **)&out, (size_t)rows * E * 4));
    CUDA_CHECK(cudaMalloc((void **)&kc, kv * 2)); CUDA_CHECK(cudaMalloc((void **)&vc, kv * 2)); CUDA_CHECK(cudaMalloc((void **)&tab_exp, 131072));
    CUDA_CHECK(cudaMalloc((void **)&st, sizeof(DeviceState))); CUDA_CHECK(cudaMalloc((void **)&slots, (size_t)rows * sizeof(SessionSlot)));
    CUDA_CHECK(cudaMemcpy(q, q_host, (size_t)rows * E * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(kc, k_host, kv * 2, cudaMemcpyHostToDevice)); CUDA_CHECK(cudaMemcpy(vc, v_host, kv * 2, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(tab_exp, te.data(), 131072, cudaMemcpyHostToDevice));
    DeviceState h_st{}; h_st.n_past = pos[0];
    CUDA_CHECK(cudaMemcpy(st, &h_st, sizeof(DeviceState), cudaMemcpyHostToDevice));
    std::vector<SessionSlot> h_slots((size_t)rows);
    for (int t = 0; t < rows; ++t) { SessionSlot &s = h_slots[(size_t)t]; s = SessionSlot{}; s.n_past = pos[t]; s.kcache = kc; s.vcache = vc; s.state = st; }
    CUDA_CHECK(cudaMemcpy(slots, h_slots.data(), (size_t)rows * sizeof(SessionSlot), cudaMemcpyHostToDevice));
    attn_smem(n_ctx);
    const dim3 ag((unsigned)n_head, (unsigned)rows);
    if (path == 1) attn_sessions_kernel<<<ag, 256, (size_t)n_ctx * 6>>>(q, slots, 0, out, E, n_ctx, kq_scale, tab_exp);
    else attn_kernel<<<ag, 256, (size_t)n_ctx * 6>>>(q, kc, vc, out, st, E, n_ctx, kq_scale, tab_exp);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(cudaMemcpy(out_host, out, (size_t)rows * E * 4, cudaMemcpyDeviceToHost));
    for (void *p : {(void *)q, (void *)out, (void *)kc, (void *)vc, (void *)tab_exp, (void *)st, (void *)slots}) cudaFree(p);
    return true;
}

void LlamaDevice::ensure_sampler() {
    if (smp_) return;
    smp_.reset(new SamplerScratch(d_.n_vocab, d_.n_ctx));
    owned_bytes_ += smp_->bytes;
}

// the columns of one kind in a step's sampling launch (the chain with greedy and constrained columns, or mirostat), in slot order: each
// column's SampleCtx carries its slot, and its StopArgsN / ConsArgsN entries follow it
struct SampleLaunch {
    smp::SampleArgsN<LlamaDevice::kMaxBatch> a{};
    smp::StopArgsN<LlamaDevice::kMaxBatch> s{};
    smp::ConsArgsN<LlamaDevice::kMaxBatch> k{};
    int n = 0;
    bool mirostat = false;   // the mirostat kernel (every column's args.mirostat is 1 or 2)
    bool cons = false;       // the constrained kernel, which takes every column's constraint table
};
template <int N>
static void launch_sample(const smp::SampleArgsN<N> &a, const smp::StopArgsN<N> &sa, const smp::ConsArgsN<N> &k, int n, bool mirostat, bool cons,
                          bool stop, cudaStream_t s) {
    using Stop = smp::StopArgsN<N>;
    if (cons && stop) smp::sample_cons_kernel<N, Stop><<<n, smp::kThreads, 0, s>>>(a, sa, k);
    else if (cons) smp::sample_cons_kernel<N><<<n, smp::kThreads, 0, s>>>(a, k);
    else if (mirostat && stop) smp::sample_kernel<N, true, Stop><<<n, smp::kThreads, 0, s>>>(a, sa);
    else if (mirostat) smp::sample_kernel<N, true><<<n, smp::kThreads, 0, s>>>(a);
    else if (stop) smp::sample_kernel<N, false, Stop><<<n, smp::kThreads, 0, s>>>(a, sa);
    else smp::sample_kernel<N, false><<<n, smp::kThreads, 0, s>>>(a);
}
// one sampling step of K's columns in one launch (grid K.n) of the kernel of its kind; stop: sample_until's step, which takes K.s.  Up to
// 8 columns the launch takes the 8-column tables, the first 8 columns of those of K's that the kernel reads.
static void launch_sample(const SampleLaunch &K, bool stop, cudaStream_t s) {
    if (K.n > 8) return launch_sample(K.a, K.s, K.k, K.n, K.mirostat, K.cons, stop, s);
    smp::SampleArgsN<8> a{};
    memcpy(a.c, K.a.c, sizeof(a.c));
    a.n_vocab = K.a.n_vocab; a.step = K.a.step;
    smp::StopArgsN<8> sa{};
    if (stop) { memcpy(sa.r, K.s.r, sizeof(sa.r)); memcpy(sa.snap, K.s.snap, sizeof(sa.snap)); sa.tab = K.s.tab; }
    smp::ConsArgsN<8> k{};
    if (K.cons) memcpy(k.c, K.k.c, sizeof(k.c));
    launch_sample(a, sa, k, K.n, K.mirostat, K.cons, stop, s);
}
// the columns of `all` by kind: kind[0] the chain, greedy and constrained columns, kind[1] mirostat
static void split_kinds(const SampleLaunch &all, SampleLaunch kind[2]) {
    for (int i = 0; i < all.n; ++i) {
        SampleLaunch &K = kind[all.a.c[i].args.mirostat ? 1 : 0];
        K.a.c[K.n] = all.a.c[i]; K.s.r[K.n] = all.s.r[i]; K.s.snap[K.n] = all.s.snap[i]; K.k.c[K.n] = all.k.c[i];
        K.cons = K.cons || all.k.c[i].off;
        ++K.n;
    }
    for (int m = 0; m < 2; ++m) { kind[m].a.n_vocab = all.a.n_vocab; kind[m].s.tab = all.s.tab; kind[m].mirostat = m == 1; }
}
// the sampling launches of step t: one per kind present
static void launch_kinds(SampleLaunch kind[2], int t, bool stop, cudaStream_t s) {
    for (int m = 0; m < 2; ++m) {
        if (!kind[m].n) continue;
        kind[m].a.step = t;
        launch_sample(kind[m], stop, s);
    }
}
// the bytes of a context's sampler state that a call moves: the generator, and μ after it with mirostat
static size_t sampler_state_bytes(const SamplingArgs &p) { return 625 * 4 + (p.mirostat ? sizeof(MirostatState) : 0); }

cudaStream_t LlamaDevice::begin_sampling(LlamaDevice *const *c, int n, const int *n_past, const SamplingArgs *p, uint32_t (*rng)[625], MirostatState *mu,
                                         const SampleConstraint *cons, SampleLaunch &all) {
    LlamaDevice &L0 = *c[0];
    smp::SampleArgsN<kMaxBatch> &a = all.a;
    a.n_vocab = L0.d_.n_vocab;
    all.n = n;
    const cudaStream_t s = n >= 2 ? open_batch(c, n, nullptr, n_past) : L0.stream_;
    for (int i = 0; i < n; ++i) {
        LlamaDevice &L = *c[i];
        L.ensure_sampler();
        SessionSlot *slot = n >= 2 ? L0.group_->slots + i : nullptr;
        a.c[i] = L.smp_->ctx(L.logits_, L.state_, slot, n_past[i]);
        a.c[i].args = p[i];
        if (p[i].temp > 0.f) {
            memcpy(L.smp_->h_rng, rng[i], 625 * 4);
            if (p[i].mirostat) *L.smp_->h_mu = mu[i];
            CUDA_CHECK(cudaMemcpyAsync(L.smp_->mt, L.smp_->h_rng, sampler_state_bytes(p[i]), cudaMemcpyHostToDevice, s));
        }
        if (cons && cons[i].off) {
            *L.smp_->h_cons = cons[i].state;
            CUDA_CHECK(cudaMemcpyAsync(L.smp_->cons, L.smp_->h_cons, sizeof(int), cudaMemcpyHostToDevice, s));
            all.k.c[i] = smp::ConsCol{cons[i].off, cons[i].tr, L.smp_->cons};
        }
    }
    return s;
}

void LlamaDevice::decode_columns(LlamaDevice *const *c, int n, int n_past, cudaStream_t s) {
    LlamaDevice &L0 = *c[0];
    CUDA_CHECK(cudaGetLastError());
    if (n == 1) L0.decode_step(-1, n_past);
    else {
        CUDA_CHECK(cudaGraphLaunch(L0.group_->graph[n], s));
        L0.launches_ += (unsigned long long)L0.group_->graph_kernels[n];
    }
}

// steps issued kReplyChunk at a time on s, at most `steps`: step(t) issues step t, and after each chunk j flags(j % 2) queues the copy of
// its done flags and ev[j % 2] is recorded.  Before chunk j >= 2 the host waits for chunk j - 2's flags (chunk j - 1 keeps the device busy
// meanwhile) and issues no more once done(j % 2) reads from them that every context is done.  Returns the steps issued.
template <class Step, class Flags, class Done>
static int issue_chunks(int steps, cudaStream_t s, const cudaEvent_t ev[2], Step step, Flags flags, Done done) {
    int issued = 0;
    for (int j = 0; issued < steps; ++j) {
        if (j >= 2) {
            CUDA_CHECK(cudaEventSynchronize(ev[j % 2]));
            if (done(j % 2)) break;
        }
        for (const int end = std::min(steps, issued + LlamaDevice::kReplyChunk); issued < end; ++issued) step(issued);
        flags(j % 2);
        CUDA_CHECK(cudaEventRecord(ev[j % 2], s));
    }
    return issued;
}

// after `steps` steps: the fed ids, generators and μ to the host, one synchronisation; returns the device ms since ev0_
float LlamaDevice::end_sampling(LlamaDevice *const *c, int n, int steps, const SamplingArgs *p, uint32_t (*rng)[625], MirostatState *mu, int32_t *ids_out,
                                cudaStream_t s) {
    LlamaDevice &L0 = *c[0];
    CUDA_CHECK(cudaEventRecord(L0.ev1_, s));
    for (int i = 0; i < n; ++i) {
        LlamaDevice &L = *c[i];
        CUDA_CHECK(cudaMemcpyAsync(L.smp_->h_ids, L.smp_->ids, (size_t)steps * 4, cudaMemcpyDeviceToHost, s));
        if (p[i].temp > 0.f) CUDA_CHECK(cudaMemcpyAsync(L.smp_->h_rng, L.smp_->mt, sampler_state_bytes(p[i]), cudaMemcpyDeviceToHost, s));
    }
    if (n == 1) L0.sync_decode();
    else {
        CUDA_CHECK(cudaStreamSynchronize(s));
        for (int i = 0; i < n; ++i) *c[i]->h_argmax_ = L0.group_->h_ids[i];   // (as decode_batch: the greedy id of the last step)
    }
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, L0.ev0_, L0.ev1_));
    for (int i = 0; i < n; ++i) {
        LlamaDevice &L = *c[i];
        const bool sampled = p[i].temp > 0.f;
        for (int t = 0; t < steps; ++t) ids_out[(size_t)t * n + i] = L.smp_->h_ids[t];
        if (sampled) memcpy(rng[i], L.smp_->h_rng, 625 * 4);
        if (sampled && p[i].mirostat) mu[i] = *L.smp_->h_mu;
    }
    return ms;
}

float LlamaDevice::sample_steps(LlamaDevice *const *c, int n, int steps, const int *n_past, const SamplingArgs &p, uint32_t (*rng)[625],
                                MirostatState *mu, int32_t *ids_out, const SampleConstraint *cons) {
    LlamaDevice &L0 = *c[0];
    SamplingArgs ps[kMaxBatch];
    std::fill(ps, ps + n, p);
    SampleLaunch all, kind[2];   // (uniform settings: one kind, one launch a step)
    const cudaStream_t s = begin_sampling(c, n, n_past, ps, rng, mu, cons, all);
    split_kinds(all, kind);
    CUDA_CHECK(cudaEventRecord(L0.ev0_, s));
    for (int t = 0; t < steps; ++t) {
        launch_kinds(kind, t, false, s);
        ++L0.launches_;
        decode_columns(c, n, n_past[0] + t, s);
    }
    return end_sampling(c, n, steps, ps, rng, mu, ids_out, s);
}

void LlamaDevice::ensure_reply() {
    if (reply_) return;
    reply_.reset(new ReplyScratch(d_.n_vocab));
    owned_bytes_ += reply_->bytes;
}
void LlamaDevice::ensure_logprob() {
    if (logprob_) return;
    logprob_.reset(new LogprobScratch(d_.n_ctx));
    owned_bytes_ += logprob_->bytes;
}
void LlamaDevice::ensure_penalty(int n_tail) {
    if (pen_ && pen_->cap >= n_tail) return;
    if (pen_) owned_bytes_ -= pen_->bytes;   // (a longer history tail than any before: the scratch grows; the last call has synchronised)
    pen_.reset();
    pen_.reset(new PenaltyScratch(d_.n_vocab, std::max(d_.n_ctx, n_tail)));
    owned_bytes_ += pen_->bytes;
}
SharedTable::~SharedTable() {
    if (dev) cudaFree(dev);
    if (std::shared_ptr<LlamaGroup> g = group.lock()) g->batch_bytes -= bytes;
}
std::shared_ptr<SharedTable> LlamaDevice::upload_table(const void *host, size_t bytes) {
    void *d = nullptr;
    if (cudaMalloc(&d, std::max<size_t>(bytes, 1)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    CUDA_CHECK(cudaMemcpy(d, host, bytes, cudaMemcpyHostToDevice));
    std::shared_ptr<SharedTable> t = std::make_shared<SharedTable>();
    t->dev = d; t->bytes = bytes; t->group = group_;
    group_->batch_bytes += bytes;
    return t;
}
bool LlamaDevice::has_token_table() const { return group_->tokens.off != nullptr; }
void LlamaDevice::set_token_table(const std::vector<int> &off, const std::string &bytes) {
    LlamaGroup &G = *group_;
    const size_t b0 = t_dev_bytes;
    int *o = nullptr; unsigned char *b = nullptr;
    dmalloc(&o, off.size() * 4);
    dmalloc(&b, std::max<size_t>(1, bytes.size()));
    CUDA_CHECK(cudaMemcpy(o, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(b, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
    G.tokens = smp::TokenTable{o, b};
    G.batch_bytes += t_dev_bytes - b0;
}

// context i's records (steps 0 .. n_rec - 1) into the caller's layout (entry e = s * n + i); the other entries of its max_steps get -1 / NaN
static void scatter_records(const lp::Record *r, int n_rec, int i, int n, int max_steps, const LogprobRequest &q) {
    const float nan = std::numeric_limits<float>::quiet_NaN();
    for (int t = 0; t < max_steps; ++t) {
        const size_t e = (size_t)t * n + i;
        const bool has = t < n_rec;
        q.logprob[e] = has ? r[t].logprob : nan;
        if (q.rank) q.rank[e] = has ? r[t].rank : -1;
        for (int j = 0; j < q.top_n; ++j) {
            q.top_ids[e * q.top_n + j] = has ? r[t].top_id[j] : -1;
            if (q.top_logprob) q.top_logprob[e * q.top_n + j] = has ? r[t].top_lp[j] : nan;
        }
    }
}

// a context's ReplyState at the start of a call: its reply's last kStopMax bytes, the stop text, nothing fed
static void reply_init(smp::ReplyState &r, const std::string &stop, const std::string &tail) {
    memset(&r, 0, sizeof(r));
    const size_t keep = std::min(tail.size(), (size_t)smp::kStopMax);
    memcpy(r.tail, tail.data() + tail.size() - keep, keep);
    r.tail_len = (int)keep;
    memcpy(r.stop, stop.data(), stop.size());
    r.stop_len = (int)stop.size();
}

float LlamaDevice::sample_until(LlamaDevice *const *c, int n, const UntilArgs *u, const int *n_past, uint32_t (*rng)[625], MirostatState *mu,
                                const std::string *tail, int32_t *ids_out, int32_t *n_out, int32_t *stopped, const SampleConstraint *cons,
                                const LogprobRequest *rec) {
    LlamaDevice &L0 = *c[0];
    SamplingArgs p[kMaxBatch]{};
    int S = 0;   // the longest budget: the most steps the call runs
    for (int i = 0; i < n; ++i) { p[i] = u[i].p; S = std::max(S, u[i].max_steps); }
    SampleLaunch all, kind[2];
    const cudaStream_t s = begin_sampling(c, n, n_past, p, rng, mu, cons, all);
    smp::StopArgsN<kMaxBatch> &sa = all.s;
    sa.tab = L0.group_->tokens;
    lp::LogprobArgs la{};
    pen::PenaltyArgs pa{};
    int n_pen = 0;
    for (int i = 0; i < n; ++i) {
        LlamaDevice &L = *c[i];
        L.ensure_reply();
        reply_init(*L.reply_->h_r, u[i].stop, tail[i]);
        L.reply_->h_r->budget = u[i].max_steps;
        L.reply_->h_r->by_budget = 0;
        CUDA_CHECK(cudaMemcpyAsync(L.reply_->r, L.reply_->h_r, sizeof(smp::UntilState), cudaMemcpyHostToDevice, s));
        sa.r[i] = L.reply_->r; sa.snap[i] = L.reply_->snap;
        if (rec) {
            L.ensure_logprob();
            la.c[i] = lp::LogprobCol{L.logits_, L.state_, L.reply_->r, L.logprob_->rec};
        }
        if (!u[i].q.neutral()) {   // the history's last repeat_last_n ids go up once; the step's sampling reads the penalised row
            const int n_last = u[i].last_ids ? u[i].n_last : 0, T = std::min(u[i].q.repeat_last_n, n_last);
            L.ensure_penalty(T);
            if (T > 0) {
                memcpy(L.pen_->h_tail, u[i].last_ids + (n_last - T), (size_t)T * 4);
                CUDA_CHECK(cudaMemcpyAsync(L.pen_->tail, L.pen_->h_tail, (size_t)T * 4, cudaMemcpyHostToDevice, s));
            }
            pa.c[n_pen++] = pen::PenaltyCol{L.logits_, L.pen_->row, L.pen_->count, L.pen_->tail, L.smp_->ids, L.state_, L.reply_->r, T, u[i].q,
                                            p[i].temp <= 0.f ? 1 : 0};
            all.a.c[i].logits = L.pen_->row;
        }
    }
    la.n_vocab = L0.d_.n_vocab; la.top_n = rec ? rec->top_n : 0;
    pa.n_vocab = L0.d_.n_vocab;
    split_kinds(all, kind);
    ReplyScratch &R0 = *L0.reply_;
    CUDA_CHECK(cudaEventRecord(L0.ev0_, s));
    const int issued = issue_chunks(S, s, R0.ev, [&](int t) {
        if (n_pen) {   // the rows this step samples from
            pa.step = t;
            pen::penalty_rows_kernel<<<n_pen, pen::kThreads, 0, s>>>(pa);
            ++L0.launches_;
        }
        launch_kinds(kind, t, true, s);
        ++L0.launches_;
        if (rec) {   // the logits the step sampled from, before the decode step replaces them
            la.step = t;
            lp::logprob_rows_kernel<<<n, lp::kThreads, 0, s>>>(la);
            ++L0.launches_;
        }
        decode_columns(c, n, n_past[0] + t, s);
    }, [&](int b) {
        for (int i = 0; i < n; ++i)
            CUDA_CHECK(cudaMemcpyAsync(R0.h_done + b * kMaxBatch + i, &c[i]->reply_->r->done, sizeof(int), cudaMemcpyDeviceToHost, s));
    }, [&](int b) {
        for (int i = 0; i < n; ++i) if (R0.h_done[b * kMaxBatch + i] == 0) return false;
        return true;
    });
    for (int i = 0; i < n; ++i)
        CUDA_CHECK(cudaMemcpyAsync(c[i]->reply_->h_r, c[i]->reply_->r, sizeof(smp::UntilState), cudaMemcpyDeviceToHost, s));
    const float ms = end_sampling(c, n, issued, p, rng, mu, ids_out, s);
    // a context that stopped before the last issued step gets back what its stopping step left
    for (int i = 0; i < n; ++i) {
        LlamaDevice &L = *c[i];
        const smp::UntilState &r = *L.reply_->h_r;
        n_out[i] = r.n_fed;
        if (stopped) stopped[i] = r.done != 0 && !r.by_budget ? 1 : 0;
        for (int t = r.n_fed; t < issued; ++t) ids_out[(size_t)t * n + i] = -1;
        if (r.done == 2) {
            CUDA_CHECK(cudaMemcpyAsync(L.logits_, L.reply_->snap, (size_t)L.d_.n_vocab * 4, cudaMemcpyDeviceToDevice, s));
            CUDA_CHECK(cudaMemcpyAsync(L.state_, &L.reply_->r->snap, sizeof(DeviceState), cudaMemcpyDeviceToDevice, s));
            *L.h_argmax_ = r.snap.argmax_id;
        }
        if (rec && r.n_fed > 0)
            CUDA_CHECK(cudaMemcpyAsync(L.logprob_->h_rec, L.logprob_->rec, (size_t)r.n_fed * sizeof(lp::Record), cudaMemcpyDeviceToHost, s));
    }
    CUDA_CHECK(cudaStreamSynchronize(s));
    for (int t = issued; t < S; ++t)
        for (int i = 0; i < n; ++i) ids_out[(size_t)t * n + i] = -1;
    if (rec)
        for (int i = 0; i < n; ++i) scatter_records(c[i]->logprob_->h_rec, n_out[i], i, n, S, *rec);
    return ms;
}

// the seam of the stop rule: one thread of reply_check_kernel over the ids, with this context's ReplyState and the group's table
int LlamaDevice::test_reply_stop(const int32_t *ids, int n, const std::string &stop, const std::string &tail) {
    ensure_reply();
    sync();
    reply_init(*reply_->h_r, stop, tail);
    int *d = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&d, ((size_t)n + 1) * 4));
    CUDA_CHECK(cudaMemcpyAsync(reply_->r, reply_->h_r, sizeof(smp::ReplyState), cudaMemcpyHostToDevice, stream_));
    CUDA_CHECK(cudaMemcpyAsync(d + 1, ids, (size_t)n * 4, cudaMemcpyHostToDevice, stream_));
    smp::reply_check_kernel<<<1, 1, 0, stream_>>>(reply_->r, group_->tokens, d + 1, n, d);
    CUDA_CHECK(cudaGetLastError());
    int at = -1;
    CUDA_CHECK(cudaMemcpyAsync(&at, d, 4, cudaMemcpyDeviceToHost, stream_));
    sync();
    cudaFree(d);
    return at;
}

// ------------------------------------------------------------------------------------------------
// beam search (llama_beam.cuh): contexts c[0 .. n) are the slots; every step ranks, merges and reorders on the device, then runs the
// decode step of every slot (n = 1: the context's own graph or megakernel, n >= 2: the batch graph with column ids -1).  The steps are
// issued kReplyChunk at a time, as in sample_until.
// ------------------------------------------------------------------------------------------------
void LlamaDevice::build_beam_scratch() {
    LlamaGroup &G = *group_;
    const size_t b0 = t_dev_bytes;
    dmalloc(&G.beam, sizeof(beam::BeamState));
    dmalloc(&G.beam_ids, (size_t)2 * beam::kMaxBeams * d_.n_ctx * 4);
    dmalloc(&G.beam_snap, (size_t)d_.n_vocab * 4);
    dmalloc(&G.beam_snap_state, sizeof(DeviceState));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_beam, sizeof(beam::BeamState), cudaHostAllocDefault));
    CUDA_CHECK(cudaHostAlloc((void **)&G.h_beam_done, 2 * sizeof(int), cudaHostAllocDefault));
    for (cudaEvent_t &e : G.beam_ev) CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CUDA_CHECK(cudaDeviceSynchronize());
    G.batch_bytes += t_dev_bytes - b0;
}

float LlamaDevice::beam_search(LlamaDevice *const *c, int n, int max_steps, int n0, const std::string &stop, const std::string &tail, float length_penalty,
                               std::vector<BeamHyp> &hyps) {
    LlamaDevice &L0 = *c[0];
    LlamaGroup &G = *L0.group_;
    for (int i = 0; i < n; ++i) c[i]->sync();
    if (!G.beam) L0.build_beam_scratch();
    const int V = L0.d_.n_vocab, stride = L0.d_.n_ctx;
    const int32_t argmax0 = L0.argmax();
    cudaStream_t s = L0.stream_;
    if (n >= 2) {
        int np[kMaxBeams];
        std::fill(np, np + n, n0);
        s = open_batch(c, n, nullptr, np);
        copy_state(L0, c + 1, n - 1, n0);   // every slot starts from the conversation; its rows below n0 are not written again
        CUDA_CHECK(cudaMemcpyAsync(G.beam_snap, L0.logits_, (size_t)V * 4, cudaMemcpyDeviceToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(G.beam_snap_state, L0.state_, sizeof(DeviceState), cudaMemcpyDeviceToDevice, s));
    }
    beam::BeamState &h = *G.h_beam;
    memset(&h, 0, sizeof h);
    for (int i = 0; i < beam::kMaxBeams; ++i) h.beam[i] = -1;
    h.beam[0] = 0;   // one live beam: no ids, S = 0, the reply's tail
    reply_init(h.tail[0], stop, tail);
    CUDA_CHECK(cudaMemcpyAsync(G.beam, G.h_beam, sizeof(beam::BeamState), cudaMemcpyHostToDevice, s));
    beam::BeamArgs a{};
    a.st = G.beam;
    for (int i = 0; i < n; ++i) { a.logits[i] = c[i]->logits_; a.state[i] = c[i]->state_; }
    a.slots = n >= 2 ? G.slots : nullptr;
    a.ids = G.beam_ids; a.hids = G.beam_ids + (size_t)beam::kMaxBeams * stride; a.stride = stride;
    a.n_beams = n; a.n_vocab = V; a.max_steps = max_steps; a.n0 = n0; a.length_penalty = length_penalty; a.tab = G.tokens;
    if (n == 1) { a.snap = G.beam_snap; a.snap_state = G.beam_snap_state; }   // (with 2 or more beams they hold the start)
    beam::ReorderArgs ra{};
    ra.st = G.beam;
    for (int i = 0; i < n; ++i) { ra.k[i] = (uint4 *)c[i]->kcache_; ra.v[i] = (uint4 *)c[i]->vcache_; }
    ra.row = (long long)L0.n_embd_local_ * 2 / 16; ra.plane = (long long)L0.d_.n_ctx * ra.row; ra.n_layer = L0.d_.n_layer; ra.n0 = n0;
    const dim3 rgrid((unsigned)std::max(1, 8 * L0.sm_count_ / (2 * L0.d_.n_layer)), (unsigned)(2 * L0.d_.n_layer));
    CUDA_CHECK(cudaEventRecord(L0.ev0_, s));
    issue_chunks(max_steps, s, G.beam_ev, [&](int t) {
        beam::beam_rank_kernel<<<n, beam::kRankThreads, 0, s>>>(a);
        beam::beam_merge_kernel<<<1, beam::kMergeThreads, 0, s>>>(a);
        L0.launches_ += 2;
        if (n >= 2) {
            beam::beam_reorder_kernel<<<rgrid, beam::kCopyThreads, 0, s>>>(ra);
            ++L0.launches_;
        }
        decode_columns(c, n, n0 + t, s);
    }, [&](int b) {
        CUDA_CHECK(cudaMemcpyAsync(G.h_beam_done + b, &G.beam->done, sizeof(int), cudaMemcpyDeviceToHost, s));
    }, [&](int b) { return G.h_beam_done[b] != 0; });
    CUDA_CHECK(cudaEventRecord(L0.ev1_, s));
    std::vector<int32_t> hid((size_t)n * stride);
    CUDA_CHECK(cudaMemcpyAsync(G.h_beam, G.beam, sizeof(beam::BeamState), cudaMemcpyDeviceToHost, s));
    CUDA_CHECK(cudaMemcpyAsync(hid.data(), a.hids, hid.size() * 4, cudaMemcpyDeviceToHost, s));
    for (int i = 1; i < n; ++i) {   // the other slots go back to the conversation as it was
        CUDA_CHECK(cudaMemcpyAsync(c[i]->logits_, G.beam_snap, (size_t)V * 4, cudaMemcpyDeviceToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(c[i]->state_, G.beam_snap_state, sizeof(DeviceState), cudaMemcpyDeviceToDevice, s));
    }
    if (n == 1) L0.sync_decode();
    else CUDA_CHECK(cudaStreamSynchronize(s));
    for (int i = 1; i < n; ++i) *c[i]->h_argmax_ = argmax0;
    if (n == 1 && h.done == 2) {   // one beam ran steps past its reply: back to what the reply's last step left
        CUDA_CHECK(cudaMemcpyAsync(L0.logits_, G.beam_snap, (size_t)V * 4, cudaMemcpyDeviceToDevice, s));
        CUDA_CHECK(cudaMemcpyAsync(L0.state_, G.beam_snap_state, sizeof(DeviceState), cudaMemcpyDeviceToDevice, s));
        DeviceState snap{};
        CUDA_CHECK(cudaMemcpyAsync(&snap, G.beam_snap_state, sizeof(DeviceState), cudaMemcpyDeviceToHost, s));
        CUDA_CHECK(cudaStreamSynchronize(s));
        *L0.h_argmax_ = snap.argmax_id;
    }
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, L0.ev0_, L0.ev1_));
    // H by final score descending, the earlier offered first on equal scores
    std::vector<int> order((size_t)h.n_h);
    for (int e = 0; e < h.n_h; ++e) order[(size_t)e] = e;
    std::sort(order.begin(), order.end(), [&](int x, int y) {
        return h.h[x].score != h.h[y].score ? h.h[x].score > h.h[y].score : h.h[x].seq < h.h[y].seq;
    });
    hyps.clear();
    for (int e : order) {
        const beam::Hyp &y = h.h[e];
        const int32_t *p = hid.data() + (size_t)e * stride;
        hyps.push_back(BeamHyp{std::vector<int32_t>(p, p + y.len), y.score, y.logprob, y.stopped});
    }
    return ms;
}

int LlamaDevice::test_beam_rank(const float *logits, int n_live, const float *S, int n_beams, int n_vocab, int32_t *parent, int32_t *id, float *c) {
    beam::BeamState *st = nullptr;
    float *lg = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&st, sizeof(beam::BeamState)));
    CUDA_CHECK(cudaMalloc((void **)&lg, (size_t)n_live * n_vocab * 4));
    std::unique_ptr<beam::BeamState> h(new beam::BeamState);
    memset(h.get(), 0, sizeof(beam::BeamState));
    for (int i = 0; i < beam::kMaxBeams; ++i) h->beam[i] = i < n_live ? i : -1;
    for (int i = 0; i < n_live; ++i) h->S[i] = S[i];
    CUDA_CHECK(cudaMemcpy(st, h.get(), sizeof(beam::BeamState), cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(lg, logits, (size_t)n_live * n_vocab * 4, cudaMemcpyHostToDevice));
    beam::BeamArgs a{};
    a.st = st;
    for (int i = 0; i < n_live; ++i) a.logits[i] = lg + (size_t)i * n_vocab;
    a.n_beams = n_beams; a.n_vocab = n_vocab; a.rank_only = 1;
    beam::beam_rank_kernel<<<n_live, beam::kRankThreads>>>(a);
    beam::beam_merge_kernel<<<1, beam::kMergeThreads>>>(a);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpy(h.get(), st, sizeof(beam::BeamState), cudaMemcpyDeviceToHost));
    for (int r = 0; r < h->n_sorted; ++r) { parent[r] = h->sorted[r].beam; id[r] = h->sorted[r].id; c[r] = h->sorted[r].c; }
    cudaFree(st); cudaFree(lg);
    return h->n_sorted;
}

void LlamaDevice::test_logprobs(const float *logits, int rows, int n_vocab, const int32_t *ids, const LogprobRequest &rec, float *kernel_ms) {
    float *lg = nullptr;
    DeviceState *st = nullptr;
    lp::Record *out = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&lg, (size_t)rows * n_vocab * 4));
    CUDA_CHECK(cudaMalloc((void **)&st, (size_t)rows * sizeof(DeviceState)));
    CUDA_CHECK(cudaMalloc((void **)&out, (size_t)rows * sizeof(lp::Record)));
    CUDA_CHECK(cudaMemcpy(lg, logits, (size_t)rows * n_vocab * 4, cudaMemcpyHostToDevice));
    std::vector<DeviceState> hs((size_t)rows);
    for (int r = 0; r < rows; ++r) { hs[(size_t)r] = DeviceState{}; hs[(size_t)r].tokens[0] = ids[r]; }
    CUDA_CHECK(cudaMemcpy(st, hs.data(), (size_t)rows * sizeof(DeviceState), cudaMemcpyHostToDevice));
    lp::LogprobArgs a{};
    for (int r = 0; r < rows; ++r) a.c[r] = lp::LogprobCol{lg + (size_t)r * n_vocab, st + r, nullptr, out + r};
    a.n_vocab = n_vocab; a.step = 0; a.top_n = rec.top_n;
    lp::logprob_rows_kernel<<<rows, lp::kThreads>>>(a);
    CUDA_CHECK(cudaGetLastError());
    if (kernel_ms) {
        constexpr int kReps = 50;
        cudaEvent_t e0, e1;
        CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
        CUDA_CHECK(cudaEventRecord(e0, 0));
        for (int i = 0; i < kReps; ++i) lp::logprob_rows_kernel<<<rows, lp::kThreads>>>(a);
        CUDA_CHECK(cudaEventRecord(e1, 0));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        *kernel_ms = ms / kReps;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    std::vector<lp::Record> h((size_t)rows);
    CUDA_CHECK(cudaMemcpy(h.data(), out, (size_t)rows * sizeof(lp::Record), cudaMemcpyDeviceToHost));
    for (int r = 0; r < rows; ++r) scatter_records(h.data() + r, 1, 0, 1, 1, LogprobRequest{rec.top_n, rec.logprob + r, rec.rank ? rec.rank + r : nullptr,
                                                                                  rec.top_ids ? rec.top_ids + (size_t)r * rec.top_n : nullptr,
                                                                                  rec.top_logprob ? rec.top_logprob + (size_t)r * rec.top_n : nullptr});
    for (void *p : {(void *)lg, (void *)st, (void *)out}) cudaFree(p);
}

void LlamaDevice::test_penalize(const float *logits, int rows, int n_vocab, const int32_t *last_ids, const int32_t *n_last, const PenaltyParams &q,
                                float *out, float *kernel_ms) {
    const size_t V = (size_t)n_vocab;
    std::vector<int> off((size_t)rows + 1, 0), T((size_t)rows);
    for (int r = 0; r < rows; ++r) {
        T[(size_t)r] = std::min(q.repeat_last_n, n_last[r]);
        off[(size_t)r + 1] = off[(size_t)r] + T[(size_t)r];
    }
    std::vector<int> tails((size_t)std::max(1, off[(size_t)rows]));
    size_t h = 0;
    for (int r = 0; r < rows; ++r) {
        std::copy(last_ids + h + (n_last[r] - T[(size_t)r]), last_ids + h + n_last[r], tails.begin() + off[(size_t)r]);
        h += (size_t)n_last[r];
    }
    float *lg = nullptr, *row = nullptr;
    int *count = nullptr, *tail = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&lg, (size_t)rows * V * 4));
    CUDA_CHECK(cudaMalloc((void **)&row, (size_t)rows * V * 4));
    CUDA_CHECK(cudaMalloc((void **)&count, (size_t)rows * V * 4));
    CUDA_CHECK(cudaMalloc((void **)&tail, tails.size() * 4));
    CUDA_CHECK(cudaMemcpy(lg, logits, (size_t)rows * V * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemset(count, 0, (size_t)rows * V * 4));
    CUDA_CHECK(cudaMemcpy(tail, tails.data(), tails.size() * 4, cudaMemcpyHostToDevice));
    pen::PenaltyArgs a{};
    for (int r = 0; r < rows; ++r)
        a.c[r] = pen::PenaltyCol{lg + r * V, row + r * V, count + r * V, tail + off[(size_t)r], nullptr, nullptr, nullptr, T[(size_t)r], q, 0};
    a.n_vocab = n_vocab; a.step = 0;
    pen::penalty_rows_kernel<<<rows, pen::kThreads>>>(a);
    CUDA_CHECK(cudaGetLastError());
    if (kernel_ms) {
        constexpr int kReps = 50;
        cudaEvent_t e0, e1;
        CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
        CUDA_CHECK(cudaEventRecord(e0, 0));
        for (int i = 0; i < kReps; ++i) pen::penalty_rows_kernel<<<rows, pen::kThreads>>>(a);
        CUDA_CHECK(cudaEventRecord(e1, 0));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        *kernel_ms = ms / kReps;
        cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
    CUDA_CHECK(cudaMemcpy(out, row, (size_t)rows * V * 4, cudaMemcpyDeviceToHost));
    for (void *p : {(void *)lg, (void *)row, (void *)count, (void *)tail}) cudaFree(p);
}

void LlamaDevice::test_sample(const float *logits, int n_vocab, const SamplingArgs &p, const uint32_t *rng, int n_draws, int32_t *out, float *kernel_ms,
                              float *mu_out) {
    SamplerScratch ss(n_vocab, n_draws);
    float *lg = nullptr, *mu_d = nullptr; DeviceState *st = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&lg, (size_t)n_vocab * 4));
    CUDA_CHECK(cudaMalloc((void **)&st, sizeof(DeviceState))); CUDA_CHECK(cudaMemset(st, 0, sizeof(DeviceState)));
    CUDA_CHECK(cudaMemcpy(lg, logits, (size_t)n_vocab * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(ss.mt, rng, 625 * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemset(ss.mu, 0, sizeof(MirostatState)));
    if (mu_out && p.mirostat) CUDA_CHECK(cudaMalloc((void **)&mu_d, (size_t)n_draws * 4));
    SampleLaunch K;
    K.a.n_vocab = n_vocab;
    K.a.c[0] = ss.ctx(lg, st, nullptr, 0);
    K.a.c[0].args = p;
    K.n = 1;
    K.mirostat = p.mirostat != 0;
    cudaEvent_t e0, e1;
    CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
    CUDA_CHECK(cudaEventRecord(e0, 0));
    for (int i = 0; i < n_draws; ++i) {
        K.a.step = i;
        launch_sample(K, false, 0);
        CUDA_CHECK(cudaGetLastError());
        if (mu_d) CUDA_CHECK(cudaMemcpyAsync(mu_d + i, &ss.mu->mu[p.mirostat - 1], 4, cudaMemcpyDeviceToDevice, 0));
    }
    CUDA_CHECK(cudaEventRecord(e1, 0));
    CUDA_CHECK(cudaDeviceSynchronize());
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    if (kernel_ms) *kernel_ms = n_draws > 0 ? ms / (float)n_draws : 0.f;
    CUDA_CHECK(cudaMemcpy(out, ss.ids, (size_t)n_draws * 4, cudaMemcpyDeviceToHost));
    if (mu_d) CUDA_CHECK(cudaMemcpy(mu_out, mu_d, (size_t)n_draws * 4, cudaMemcpyDeviceToHost));
    cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(lg); cudaFree(st); cudaFree(mu_d);
}

void LlamaDevice::test_libm(int fn, uint32_t lo, uint32_t n, float *out_host, float x) {
    float *d = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&d, (size_t)n * 4));
    if (fn <= 1) smp::libm_kernel<<<1024, 256>>>(fn, lo, n, d);
    else smp::mirostat_libm_kernel<<<1024, 256>>>(fn - 2, x, lo, n, d);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaMemcpy(out_host, d, (size_t)n * 4, cudaMemcpyDeviceToHost));
    cudaFree(d);
}

}  // namespace mg4

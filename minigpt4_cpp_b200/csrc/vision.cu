// vision.cu — host side of the vision graph (see vision.h, vision_kernels.cuh).
#include "vision.h"
#include <functional>
#include "vision_kernels.cuh"
#include <math.h>
#include <string.h>
#include <algorithm>

namespace mg4 {
using namespace vk;

struct GemmPlan { CUtensorMap tmW, tmX; GemmArgs a; size_t smem; int grid; int grid_y; int grid_z; };  // grid_y > 1: token split; grid_z > 1: + split-K

// ---- TMA descriptor encoding through the driver entry point (no libcuda link dependency) ----------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                                  const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr; cudaDriverEntryPointQueryResult qr;
        CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
        if (!p || qr != cudaDriverEntryPointSuccess) MG4_PANIC("cuTensorMapEncodeTiled is not available from this driver");
        fn = (EncodeTiledFn)p;
    }
    return fn;
}
static void make_map_f16(CUtensorMap *m, const void *ptr, int rows, int cols, int box_rows) {
    cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
    cuuint32_t es[2] = {1, 1};
    CUresult r = encode_fn()(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, (void *)ptr, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) MG4_PANIC("cuTensorMapEncodeTiled failed (%d) for [%d x %d] box %d", (int)r, rows, cols, box_rows);
}

static const int kTokTiles[] = {32, 80, 144, 256};   // instantiated token tiles (wgmma N) of gemm_f16_wgmma
static int tok_tile(int t) { for (int nt : kTokTiles) if (t <= nt) return nt; return 256; }

static bool gemm_shape_ok(int M, int K, int T) { return M > 0 && K > 0 && M % 128 == 0 && K % 64 == 0 && T >= 1 && T <= 272; }
// tsplit: split the tokens of the T > 128 GEMMs over grid.y (load(): unless MINIGPT4_B200_VISION_TSPLIT=0)
static GemmPlan *make_plan(const __half *W, int M, int K, const __half *X, int T, int epi, bool tsplit, int ksplit = 1) {
    if (!gemm_shape_ok(M, K, T)) MG4_PANIC("gemm plan: unsupported shape M=%d K=%d T=%d", M, K, T);
    GemmPlan *p = new GemmPlan();
    memset(p, 0, sizeof(*p));
    GemmArgs &a = p->a;
    a.M_out = M; a.T = T; a.K = K; a.epi = epi;
    p->grid = M / 128;
    p->grid_z = 1;
    int splits = 1;
    // split the tokens of the 257-token GEMMs over grid.y CTAs so that most of the 132 SMs work (tsplit false: as few CTAs per weight slab as fit)
    if (tsplit && T > 128 && epi != GE_PATCH) {
        splits = std::max(2, std::min(4, 132 / p->grid));                      // 33 tiles -> 4 (132 CTAs), 48 -> 2 (96), 11 / 12 -> 4 (x split-K)
        if (ksplit > 1 && ksplit <= K / 64) {                                  // split-K: grid.z slices of whole k-blocks, raw partials out (GE_PARTIAL)
            a.k_split_blocks = (K / 64 + ksplit - 1) / ksplit;
            p->grid_z = (K / 64 + a.k_split_blocks - 1) / a.k_split_blocks;
            if (p->grid_z > 1) a.epi = GE_PARTIAL; else { a.k_split_blocks = 0; p->grid_z = 1; }
        }
    }
    a.nt = tok_tile((T + splits - 1) / splits);                                // tokens per CTA
    p->grid_y = (T + a.nt - 1) / a.nt;
    a.stage_bytes = 16384 + a.nt * 128;                                        // a multiple of 1024 (128-byte-swizzle atoms)
    a.stages = std::min(8, (200 * 1024) / a.stage_bytes);
    p->smem = (size_t)a.stages * a.stage_bytes + 1024 + 256;
    make_map_f16(&p->tmW, W, M, K, 128);
    make_map_f16(&p->tmX, X, T, K, a.nt);
    return p;
}
template <int NT> static void launch_gemm(const GemmPlan *p, cudaStream_t s) {
    static bool configured[64] = {};   // per device
    int dev = 0; cudaGetDevice(&dev);
    if (!configured[dev & 63]) {
        CUDA_CHECK(cudaFuncSetAttribute(gemm_f16_wgmma<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 210 * 1024));
        configured[dev & 63] = true;
    }
    gemm_f16_wgmma<NT><<<dim3((unsigned)p->grid, (unsigned)p->grid_y, (unsigned)p->grid_z), kGemmThreads, p->smem, s>>>(p->tmW, p->tmX, p->a);
}
static void launch_plan(const GemmPlan *p, cudaStream_t s) {
    switch (p->a.nt) {
        case 32: launch_gemm<32>(p, s); break;
        case 80: launch_gemm<80>(p, s); break;
        case 144: launch_gemm<144>(p, s); break;
        case 256: launch_gemm<256>(p, s); break;
        default: MG4_PANIC("gemm plan: token tile %d is not instantiated", p->a.nt);
    }
    CUDA_CHECK(cudaGetLastError());
}

static inline unsigned short f2h_bits(float f) { __half h = __float2half_rn(f); unsigned short u; memcpy(&u, &h, 2); return u; }
static inline float h2f_bits(unsigned short u) { __half h; memcpy(&h, &u, 2); return __half2float(h); }
static __half *upload_table(int which) {  // ggml's fp16 LUTs (ggml_init): 0 = gelu (tanh form), 1 = exp
    std::vector<unsigned short> t(65536);
    for (int i = 0; i < 65536; ++i) {
        const float x = h2f_bits((unsigned short)i);
        const float y = which == 0 ? 0.5f * x * (1.0f + tanhf(0.79788456080286535587989211986876f * x * (1.0f + 0.044715f * x * x))) : expf(x);
        t[(size_t)i] = f2h_bits(y);
    }
    __half *d; CUDA_CHECK(cudaMalloc((void **)&d, 131072)); CUDA_CHECK(cudaMemcpy(d, t.data(), 131072, cudaMemcpyHostToDevice));
    return d;
}

// ------------------------------------------------------------------------------------------------
VisionDevice::VisionDevice() {}
VisionDevice::~VisionDevice() {
    if (graph_) cudaGraphExecDestroy(graph_);
    for (GemmPlan *p : plans_) delete p;
    for (void *p : allocs_) cudaFree(p);
    if (h_out_) cudaFreeHost(h_out_);
    if (h_img_) cudaFreeHost(h_img_);
    if (ev0_) cudaEventDestroy(ev0_);
    if (ev1_) cudaEventDestroy(ev1_);
    if (stream_) cudaStreamDestroy(stream_);
}
void *VisionDevice::dalloc(size_t n) {
    void *p; CUDA_CHECK(cudaMalloc(&p, n)); CUDA_CHECK(cudaMemset(p, 0, n)); allocs_.push_back(p); return p;
}
// Every >= 2-D weight ends up as an F16 row-major operand of the tensor-core GEMMs.  F16 containers (the reference's convert.py
// output) are copied as they are.  Quantised containers (minigpt4_quantize_model output: the README's pre-quantised downloads) and
// F32 ones are expanded to F16 once, here, on the device.  NOTE (numerics): ggml would run such a matrix through its quantised
// mul_mat (activations quantised to Q8_0/Q8_1, integer block dots); here the weight's dequantised value, rounded to F16, meets the
// F16-rounded activation on the tensor cores.  Both are faithful to the stored weights to ~1e-3; the parity test bounds the
// difference on the final embedding (tests/test_quantized_vision_gpu.py).
static bool vision_type_ok(int gg) { return gg == GG_F16 || gg == GG_F32 || gg == GG_Q4_0 || gg == GG_Q4_1 || gg == GG_Q5_0 || gg == GG_Q5_1 || gg == GG_Q8_0; }
void VisionDevice::put16(const HostTensor &t, __half *dst) {
    if (!vision_type_ok(t.gg)) MG4_PANIC("tensor %s: ggml type %d is not supported by the vision graph (F16, F32, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0)", t.name.c_str(), t.gg);
    const size_t n = (size_t)t.nelements();
    if (t.gg == GG_F16) { CUDA_CHECK(cudaMemcpy(dst, t.data, n * 2, cudaMemcpyHostToDevice)); return; }
    unsigned char *raw = nullptr;
    CUDA_CHECK(cudaMalloc((void **)&raw, t.nbytes));
    CUDA_CHECK(cudaMemcpy(raw, t.data, t.nbytes, cudaMemcpyHostToDevice));
    dequant_to_f16_kernel<<<(unsigned)((n + 255) / 256), 256>>>(t.gg, raw, n, dst);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaDeviceSynchronize());
    cudaFree(raw);
}
// Weights live once per model: a lane created for batched encoding (Engine::encode_images) finds every weight of the first lane under its key
// and only allocates its own activations, plans and graph.
void *VisionDevice::cached(const std::string &key, size_t bytes, const std::function<void(void *)> &fill) {
    auto it = wcache_->find(key);
    if (it != wcache_->end()) { weight_bytes_ += bytes; return it->second; }
    void *d = dalloc(bytes);
    fill(d);
    (*wcache_)[key] = d;
    weight_bytes_ += bytes;
    return d;
}
const __half *VisionDevice::w16(const VisionFile &f, const std::string &model, const std::string &name, int rows, int cols) {
    const HostTensor &t = f.get(model, name);
    if (t.nelements() != (int64_t)rows * cols) MG4_PANIC("tensor %s.%s: expected %d x %d", model.c_str(), name.c_str(), rows, cols);
    return (const __half *)cached("h:" + model + "/" + name, (size_t)rows * cols * 2, [&](void *d) { put16(t, (__half *)d); });
}
const float *VisionDevice::w32(const VisionFile &f, const std::string &model, const std::string &name, int n) {
    const HostTensor &t = f.get(model, name);
    if (t.gg != GG_F32 || t.nelements() != n) MG4_PANIC("tensor %s.%s: expected %d F32 values", model.c_str(), name.c_str(), n);
    return (const float *)cached("f:" + model + "/" + name, t.nbytes, [&](void *d) { CUDA_CHECK(cudaMemcpy(d, t.data, t.nbytes, cudaMemcpyHostToDevice)); });
}

Error VisionDevice::load(const VisionFile &f, const VisionDevice *share) {
    wcache_ = share ? share->wcache_ : std::make_shared<std::map<std::string, void *>>();
    long v = 0;
    if (json_find_int(f.config_json, "Qformer", "encoder_width", &v)) d_.D = (int)v;
    if (json_find_int(f.config_json, "Qformer", "query_length", &v)) d_.n_q = (int)v;
    const HostTensor &pos = f.get("visual_encoder", "pos_embed");
    d_.T = (int)pos.ne[1];
    d_.H = d_.D / 88; d_.dh = 88;
    // the kernels take D = 16 heads of 88 (attention_f32_kernel<88>), D <= 1536 (12 values per LayerNorm thread) and D % 128 == 0 (GEMM
    // tiles): in practice D = 1408, EVA ViT-g
    if (d_.D != (int)pos.ne[0] || d_.D % 128 || d_.D % 88 || d_.D > 1536 || d_.T != 257 || d_.n_q != 32) { MG4_ERR("unsupported vision geometry D=%d T=%d queries=%d", d_.D, d_.T, d_.n_q); return ErrLoadModelFileHeader; }
    d_.n_blocks = 0; while (f.find("visual_encoder", "blocks." + std::to_string(d_.n_blocks) + ".norm1.weight")) ++d_.n_blocks;
    d_.q_layers = 0; while (f.find("Qformer", "bert.encoder.layer." + std::to_string(d_.q_layers) + ".attention.self.query.weight")) ++d_.q_layers;
    if (json_find_int(f.config_json, "Qformer", "num_hidden_layers", &v) && (int)v < d_.q_layers) d_.q_layers = (int)v;  // reference loops num_hidden_layers (:2293)
    const HostTensor &lp = f.get("llama_proj", "weight");
    d_.n_embd_llm = (int)lp.ne[1];
    if (d_.n_embd_llm != 4096 && d_.n_embd_llm != 5120) { MG4_ERR("llama_proj width %d is neither 7B nor 13B", d_.n_embd_llm); return ErrLoadModelFileHeader; }
    d_.FF = (int)f.get("visual_encoder", "blocks.0.mlp.fc1.weight").ne[1];
    const int D = d_.D, T = d_.T, FF = d_.FF, QH = 768, NQ = 32;

    CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    CUDA_CHECK(cudaEventCreate(&ev0_)); CUDA_CHECK(cudaEventCreate(&ev1_));
    tab_gelu_ = (__half *)cached("tab:gelu", 131072, [&](void *d) { __half *t = upload_table(0); CUDA_CHECK(cudaMemcpy(d, t, 131072, cudaMemcpyDeviceToDevice)); cudaFree(t); });
    tab_exp_ = (__half *)cached("tab:exp", 131072, [&](void *d) { __half *t = upload_table(1); CUDA_CHECK(cudaMemcpy(d, t, 131072, cudaMemcpyDeviceToDevice)); cudaFree(t); });
    weight_bytes_ = 0;

    // activations
    img_ = (float *)dalloc((size_t)3 * 224 * 224 * 4);
    patches_ = (__half *)dalloc((size_t)256 * 640 * 2);
    x_ = (float *)dalloc((size_t)T * D * 4);
    // proj / fc2 as n split-K slices (default 3; MINIGPT4_B200_VISION_SPLITK=1 turns it off for A/B runs) whose partial
    // sums the following LayerNorm folds into x in slice order
    const bool tsplit = !(getenv("MINIGPT4_B200_VISION_TSPLIT") && atoi(getenv("MINIGPT4_B200_VISION_TSPLIT")) == 0);
    splitk_ = !tsplit ? 1 : getenv("MINIGPT4_B200_VISION_SPLITK") ? std::max(1, std::min(4, atoi(getenv("MINIGPT4_B200_VISION_SPLITK")))) : 3;
    parts_ = splitk_ > 1 ? (float *)dalloc((size_t)splitk_ * T * D * 4) : nullptr;
    ln16_ = (__half *)dalloc((size_t)T * D * 2);
    qkv_ = (float *)dalloc((size_t)T * 3 * D * 4);
    ctx16_ = (__half *)dalloc((size_t)T * D * 2);
    h16_ = (__half *)dalloc((size_t)T * FF * 2);
    img_emb16_ = (__half *)dalloc((size_t)T * D * 2);
    hs_ = (float *)dalloc((size_t)NQ * QH * 4); hs16_ = (__half *)dalloc((size_t)NQ * QH * 2);
    qa_ = (float *)dalloc((size_t)NQ * QH * 4); qa16_ = (__half *)dalloc((size_t)NQ * QH * 2);
    qc_ = (float *)dalloc((size_t)NQ * QH * 4); qc16_ = (__half *)dalloc((size_t)NQ * QH * 2);
    qqkv_ = (float *)dalloc((size_t)NQ * 3 * QH * 4);
    qq_ = (float *)dalloc((size_t)NQ * QH * 4);
    qkv_cross_ = (float *)dalloc((size_t)T * 2 * QH * 4);
    qctx16_ = (__half *)dalloc((size_t)NQ * QH * 2);
    qh16_ = (__half *)dalloc((size_t)NQ * 3072 * 2);
    proj_out_ = (float *)dalloc((size_t)NQ * d_.n_embd_llm * 4);
    float *qtmp = (float *)dalloc((size_t)NQ * QH * 4);
    CUDA_CHECK(cudaHostAlloc((void **)&h_out_, (size_t)NQ * d_.n_embd_llm * 4, cudaHostAllocDefault));
    CUDA_CHECK(cudaHostAlloc((void **)&h_img_, (size_t)3 * 224 * 224 * 4, cudaHostAllocDefault));

    auto add_plan = [&](GemmPlan *p) { plans_.push_back(p); flops_ += 2.0 * p->a.M_out * p->a.T * p->a.K; return p; };
    const std::string VE = "visual_encoder";
    cls_ = w32(f, VE, "cls_token", D);
    pos_ = w32(f, VE, "pos_embed", T * D);
    {   // patch embedding: [D][3*14*14] -> [D][640]
        const HostTensor &pw = f.get(VE, "patch_embed.proj.weight");
        if (pw.nelements() != (int64_t)D * 588) MG4_PANIC("patch_embed.proj.weight must be [14,14,3,%d]", D);
        __half *padded = (__half *)cached("patch_embed.padded", (size_t)D * 640 * 2, [&](void *d) {
            __half *raw; CUDA_CHECK(cudaMalloc((void **)&raw, (size_t)D * 588 * 2)); put16(pw, raw);
            CUDA_CHECK(cudaMemset(d, 0, (size_t)D * 640 * 2));
            pad_rows_f16_kernel<<<(unsigned)(((size_t)D * 640 + 255) / 256), 256>>>(raw, D, 588, (__half *)d, 640);
            CUDA_CHECK(cudaDeviceSynchronize()); cudaFree(raw);
        });
        patch_ = add_plan(make_plan(padded, D, 640, patches_, 256, GE_PATCH, tsplit));
        patch_->a.bias = w32(f, VE, "patch_embed.proj.bias", D); patch_->a.out_f32 = x_; patch_->a.ld_out = D; patch_->a.pos = pos_;
    }
    blocks_.resize((size_t)d_.n_blocks);
    for (int i = 0; i < d_.n_blocks; ++i) {
        Block &b = blocks_[(size_t)i];
        const std::string p = "blocks." + std::to_string(i) + ".";
        b.n1w = w32(f, VE, p + "norm1.weight", D); b.n1b = w32(f, VE, p + "norm1.bias", D);
        b.n2w = w32(f, VE, p + "norm2.weight", D); b.n2b = w32(f, VE, p + "norm2.bias", D);
        {   // qkv_bias = [q_bias, 0, v_bias] (reference minigpt4.cpp:1259-1262)
            const HostTensor &q = f.get(VE, p + "attn.q_bias"), &vb = f.get(VE, p + "attn.v_bias");
            b.qkv_bias = (const float *)cached("qkv_bias:" + p, (size_t)3 * D * 4, [&](void *d) {
                float *qb = (float *)d;
                CUDA_CHECK(cudaMemset(qb, 0, (size_t)3 * D * 4));
                CUDA_CHECK(cudaMemcpy(qb, q.data, (size_t)D * 4, cudaMemcpyHostToDevice));
                CUDA_CHECK(cudaMemcpy(qb + 2 * D, vb.data, (size_t)D * 4, cudaMemcpyHostToDevice));
            });
        }
        b.qkv = add_plan(make_plan(w16(f, VE, p + "attn.qkv.weight", 3 * D, D), 3 * D, D, ln16_, T, GE_QSCALE, tsplit));
        b.qkv->a.bias = b.qkv_bias; b.qkv->a.qscale = 1.0f / sqrtf((float)d_.dh); b.qkv->a.qscale_rows = D; b.qkv->a.out_f32 = qkv_; b.qkv->a.ld_out = 3 * D;
        b.proj = add_plan(make_plan(w16(f, VE, p + "attn.proj.weight", D, D), D, D, ctx16_, T, GE_RESID, tsplit, splitk_));
        b.proj->a.bias = w32(f, VE, p + "attn.proj.bias", D); b.proj->a.out_f32 = x_; b.proj->a.resid = x_; b.proj->a.ld_out = D;
        b.proj->a.partial = parts_; b.proj->a.partial_stride = (long long)T * D;
        b.fc1 = add_plan(make_plan(w16(f, VE, p + "mlp.fc1.weight", FF, D), FF, D, ln16_, T, GE_GELU_F16, tsplit));
        b.fc1->a.bias = w32(f, VE, p + "mlp.fc1.bias", FF); b.fc1->a.out_f16 = h16_; b.fc1->a.ld_out = FF; b.fc1->a.tab_gelu = tab_gelu_;
        b.fc2 = add_plan(make_plan(w16(f, VE, p + "mlp.fc2.weight", D, FF), D, FF, h16_, T, GE_RESID, tsplit, splitk_));
        b.fc2->a.bias = w32(f, VE, p + "mlp.fc2.bias", D); b.fc2->a.out_f32 = x_; b.fc2->a.resid = x_; b.fc2->a.ld_out = D;
        b.fc2->a.partial = parts_; b.fc2->a.partial_stride = (long long)T * D;
        flops_ += 4.0 * d_.H * (double)T * T * d_.dh;
    }
    lnv_w_ = w32(f, "ln_vision", "weight", D); lnv_b_ = w32(f, "ln_vision", "bias", D);
    qtok_ = w32(f, "query_tokens", "weight", NQ * QH);
    const std::string QF = "Qformer";
    qln_w_ = w32(f, QF, "bert.embeddings.LayerNorm.weight", QH); qln_b_ = w32(f, QF, "bert.embeddings.LayerNorm.bias", QH);
    auto cat16 = [&](std::initializer_list<const HostTensor *> ts, int cols) {  // row-concatenate matrices as F16
        size_t total = 0; std::string key = "cat16";
        for (auto t : ts) { if (t->ne[0] != cols) MG4_PANIC("Q-Former matrix %s must have %d columns", t->name.c_str(), cols); total += (size_t)t->nelements() * 2; key += ":" + t->name; }
        return (const __half *)cached(key, total, [&](void *dv) {
            unsigned char *d = (unsigned char *)dv; size_t off = 0;
            for (auto t : ts) { put16(*t, (__half *)(d + off)); off += (size_t)t->nelements() * 2; }
        });
    };
    auto cat32 = [&](std::initializer_list<const HostTensor *> ts) {
        size_t total = 0; std::string key = "cat32";
        for (auto t : ts) { total += t->nbytes; key += ":" + t->name; }
        return (const float *)cached(key, total, [&](void *dv) {
            unsigned char *d = (unsigned char *)dv; size_t off = 0;
            for (auto t : ts) { CUDA_CHECK(cudaMemcpy(d + off, t->data, t->nbytes, cudaMemcpyHostToDevice)); off += t->nbytes; }
        });
    };
    qlayers_.resize((size_t)d_.q_layers);
    for (int i = 0; i < d_.q_layers; ++i) {
        QLayer &L = qlayers_[(size_t)i];
        const std::string p = "bert.encoder.layer." + std::to_string(i) + ".";
        L.sa_qkv = add_plan(make_plan(cat16({&f.get(QF, p + "attention.self.query.weight"), &f.get(QF, p + "attention.self.key.weight"), &f.get(QF, p + "attention.self.value.weight")}, QH),
                                      3 * QH, QH, hs16_, NQ, GE_BIAS, tsplit));
        L.sa_qkv_b = cat32({&f.get(QF, p + "attention.self.query.bias"), &f.get(QF, p + "attention.self.key.bias"), &f.get(QF, p + "attention.self.value.bias")});
        L.sa_qkv->a.bias = L.sa_qkv_b; L.sa_qkv->a.out_f32 = qqkv_; L.sa_qkv->a.ld_out = 3 * QH;
        L.sa_o = add_plan(make_plan(w16(f, QF, p + "attention.output.dense.weight", QH, QH), QH, QH, qctx16_, NQ, GE_RESID, tsplit));
        L.sa_o->a.bias = w32(f, QF, p + "attention.output.dense.bias", QH); L.sa_o->a.out_f32 = qtmp; L.sa_o->a.resid = hs_; L.sa_o->a.ld_out = QH;
        L.sa_ln_w = w32(f, QF, p + "attention.output.LayerNorm.weight", QH); L.sa_ln_b = w32(f, QF, p + "attention.output.LayerNorm.bias", QH);
        flops_ += 4.0 * 12 * NQ * NQ * 64;
        L.cross = f.find(QF, p + "crossattention.self.query.weight") != nullptr;
        if (L.cross) {
            L.ca_q = add_plan(make_plan(w16(f, QF, p + "crossattention.self.query.weight", QH, QH), QH, QH, qa16_, NQ, GE_BIAS, tsplit));
            L.ca_q->a.bias = w32(f, QF, p + "crossattention.self.query.bias", QH); L.ca_q->a.out_f32 = qq_; L.ca_q->a.ld_out = QH;
            L.ca_kv = add_plan(make_plan(cat16({&f.get(QF, p + "crossattention.self.key.weight"), &f.get(QF, p + "crossattention.self.value.weight")}, D), 2 * QH, D, img_emb16_, T, GE_BIAS, tsplit));
            L.ca_kv_b = cat32({&f.get(QF, p + "crossattention.self.key.bias"), &f.get(QF, p + "crossattention.self.value.bias")});
            L.ca_kv->a.bias = L.ca_kv_b; L.ca_kv->a.out_f32 = qkv_cross_; L.ca_kv->a.ld_out = 2 * QH;
            L.ca_o = add_plan(make_plan(w16(f, QF, p + "crossattention.output.dense.weight", QH, QH), QH, QH, qctx16_, NQ, GE_RESID, tsplit));
            L.ca_o->a.bias = w32(f, QF, p + "crossattention.output.dense.bias", QH); L.ca_o->a.out_f32 = qtmp; L.ca_o->a.resid = qa_; L.ca_o->a.ld_out = QH;
            L.ca_ln_w = w32(f, QF, p + "crossattention.output.LayerNorm.weight", QH); L.ca_ln_b = w32(f, QF, p + "crossattention.output.LayerNorm.bias", QH);
            flops_ += 4.0 * 12 * NQ * T * 64;
        }
        const int QFF = (int)f.get(QF, p + "intermediate_query.dense.weight").ne[1];
        if (QFF != 3072) MG4_PANIC("Q-Former intermediate size %d unsupported", QFF);
        L.ff1 = add_plan(make_plan(w16(f, QF, p + "intermediate_query.dense.weight", QFF, QH), QFF, QH, L.cross ? qc16_ : qa16_, NQ, GE_GELU_F16, tsplit));
        L.ff1->a.bias = w32(f, QF, p + "intermediate_query.dense.bias", QFF); L.ff1->a.out_f16 = qh16_; L.ff1->a.ld_out = QFF; L.ff1->a.tab_gelu = tab_gelu_;
        L.ff2 = add_plan(make_plan(w16(f, QF, p + "output_query.dense.weight", QH, QFF), QH, QFF, qh16_, NQ, GE_RESID, tsplit));
        L.ff2->a.bias = w32(f, QF, p + "output_query.dense.bias", QH); L.ff2->a.out_f32 = qtmp; L.ff2->a.resid = L.cross ? qc_ : qa_; L.ff2->a.ld_out = QH;
        L.ff_ln_w = w32(f, QF, p + "output_query.LayerNorm.weight", QH); L.ff_ln_b = w32(f, QF, p + "output_query.LayerNorm.bias", QH);
    }
    proj_ = add_plan(make_plan(w16(f, "llama_proj", "weight", d_.n_embd_llm, QH), d_.n_embd_llm, QH, hs16_, NQ, GE_BIAS, tsplit));
    proj_->a.bias = w32(f, "llama_proj", "bias", d_.n_embd_llm); proj_->a.out_f32 = proj_out_; proj_->a.ld_out = d_.n_embd_llm;
    qtmp_ = qtmp;

    // capture the forward as one graph
    CUDA_CHECK(cudaDeviceSynchronize());
    cudaGraph_t g = nullptr;
    launches_ = 0;
    CUDA_CHECK(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal));
    record();
    CUDA_CHECK(cudaStreamEndCapture(stream_, &g));
    CUDA_CHECK(cudaGraphInstantiate(&graph_, g, 0));
    CUDA_CHECK(cudaGraphDestroy(g));
    graph_kernels_ = (int)launches_; launches_ = 0;
    MG4_INFO("vision graph on device: %d ViT blocks, %d Q-Former layers, %.1f GFLOP/image, %.1f MB weights, %d kernels/encode", d_.n_blocks, d_.q_layers,
             flops_ * 1e-9, weight_bytes_ / 1048576.0, graph_kernels_);
    return ErrNone;
}

static size_t attn_smem(int nk, int dh) { const int nkp = (nk + 31) & ~31; return ((size_t)nk * (dh + 4) + (size_t)nk * dh + (size_t)8 * kAttnNQ * (nkp > dh ? nkp : dh)) * 4; }
static void launch_attention(int dh, dim3 grid, cudaStream_t s, const float *q, int ldq, const float *k, const float *v, int ldkv, int nq, int nk, float div, int qpc,
                             __half *out, int ld_out, const __half *tab) {
    static bool cfg[64] = {};   // per device
    int dev = 0; cudaGetDevice(&dev);
    if (!cfg[dev & 63]) {
        CUDA_CHECK(cudaFuncSetAttribute(attention_f32_kernel<88>, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024));
        CUDA_CHECK(cudaFuncSetAttribute(attention_f32_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 225 * 1024));
        cfg[dev & 63] = true;
    }
    if (nk > 288) MG4_PANIC("attention: at most 288 keys (got %d)", nk);
    const size_t sm = attn_smem(nk, dh);
    if (dh == 88) attention_f32_kernel<88><<<grid, 256, sm, s>>>(q, ldq, k, v, ldkv, nq, nk, div, qpc, out, ld_out, tab);
    else if (dh == 64) attention_f32_kernel<64><<<grid, 256, sm, s>>>(q, ldq, k, v, ldkv, nq, nk, div, qpc, out, ld_out, tab);
    else MG4_PANIC("attention: head_dim %d not instantiated", dh);
    CUDA_CHECK(cudaGetLastError());
}

// taps != null: the same sequence, eagerly, with each stage copied to the host once it is complete (encode_taps)
void VisionDevice::record(const Taps *taps) {
    const int D = d_.D, T = d_.T, QH = 768, NQ = 32;
    cudaStream_t s = stream_;
    int pending_parts = 0;  // split-K slices of the last residual GEMM that the next LayerNorm over x_ must fold in
    int pending_block = -1; // taps: block whose residual stream is complete once the next LayerNorm over x_ has folded its slices
    auto tap = [&](float *dst, const float *src, size_t n) {
        CUDA_CHECK(cudaMemcpyAsync(dst, src, n * 4, cudaMemcpyDeviceToHost, s)); CUDA_CHECK(cudaStreamSynchronize(s));
    };
    auto ln = [&](const float *x, int rows, int n, const float *w, const float *b, __half *o16, float *o32) {
        if (pending_parts > 0 && x == x_ && !o32) {
            layernorm_fold_kernel<<<rows, 128, 0, s>>>(x_, rows, n, w, b, o16, parts_, pending_parts, (long long)rows * n); pending_parts = 0;
        } else layernorm_kernel<<<rows, 128, 0, s>>>(x, rows, n, w, b, o16, o32, nullptr);
        ++launches_;
        if (taps && x == x_ && pending_block >= 0) {
            if (taps->vit_blocks) tap(taps->vit_blocks + (size_t)pending_block * T * D, x_, (size_t)T * D);
            pending_block = -1;
        }
    };
    auto gemm = [&](GemmPlan *p) { launch_plan(p, s); ++launches_; if (p->a.epi == GE_PARTIAL) pending_parts = std::max(1, p->grid_z); };

    im2col_patch_kernel<<<256, 128, 0, s>>>(img_, patches_, 640); ++launches_;
    gemm(patch_);
    cls_row_kernel<<<(D + 255) / 256, 256, 0, s>>>(cls_, pos_, x_, D); ++launches_;
    if (taps && taps->embed) tap(taps->embed, x_, (size_t)T * D);
    const int qpc = (T + 8) / 9;  // 9 query chunks per head -> 144 CTAs (one wave); 29 queries = 8 warps x 4 queries in one pass
    for (size_t i = 0; i < blocks_.size(); ++i) {
        Block &b = blocks_[i];
        ln(x_, T, D, b.n1w, b.n1b, ln16_, nullptr);
        gemm(b.qkv);
        launch_attention(d_.dh, dim3((unsigned)d_.H, (unsigned)((T + qpc - 1) / qpc)), s, qkv_, 3 * D, qkv_ + D, qkv_ + 2 * D, 3 * D, T, T, 1.0f, qpc, ctx16_, D, tab_exp_); ++launches_;
        gemm(b.proj);
        ln(x_, T, D, b.n2w, b.n2b, ln16_, nullptr);
        gemm(b.fc1);
        gemm(b.fc2);
        pending_block = (int)i;
    }
    ln(x_, T, D, lnv_w_, lnv_b_, img_emb16_, nullptr);
    if (taps && taps->ln_vision) {
        std::vector<__half> h((size_t)T * D);
        CUDA_CHECK(cudaMemcpyAsync(h.data(), img_emb16_, h.size() * 2, cudaMemcpyDeviceToHost, s)); CUDA_CHECK(cudaStreamSynchronize(s));
        for (size_t i = 0; i < h.size(); ++i) taps->ln_vision[i] = __half2float(h[i]);
    }
    ln(qtok_, NQ, QH, qln_w_, qln_b_, hs16_, hs_);
    for (size_t i = 0; i < qlayers_.size(); ++i) {
        QLayer &L = qlayers_[i];
        gemm(L.sa_qkv);
        launch_attention(64, dim3(12, 1), s, qqkv_, 3 * QH, qqkv_ + QH, qqkv_ + 2 * QH, 3 * QH, NQ, NQ, 8.0f, NQ, qctx16_, QH, tab_exp_); ++launches_;
        gemm(L.sa_o);
        ln(qtmp_, NQ, QH, L.sa_ln_w, L.sa_ln_b, qa16_, qa_);
        if (L.cross) {
            gemm(L.ca_q);
            gemm(L.ca_kv);
            launch_attention(64, dim3(12, 2), s, qq_, QH, qkv_cross_, qkv_cross_ + QH, 2 * QH, NQ, T, 8.0f, 16, qctx16_, QH, tab_exp_); ++launches_;
            gemm(L.ca_o);
            ln(qtmp_, NQ, QH, L.ca_ln_w, L.ca_ln_b, qc16_, qc_);
        }
        gemm(L.ff1);
        gemm(L.ff2);
        ln(qtmp_, NQ, QH, L.ff_ln_w, L.ff_ln_b, hs16_, hs_);
        if (taps && taps->qformer) tap(taps->qformer + i * NQ * QH, hs_, (size_t)NQ * QH);
    }
    gemm(proj_);
    CUDA_CHECK(cudaGetLastError());
    if (taps && taps->out) tap(taps->out, proj_out_, (size_t)NQ * d_.n_embd_llm);
}

void VisionDevice::encode_begin(const float *image_host) {   // asynchronous: image H2D, the graph, embedding D2H on this lane's stream
    const size_t ib = (size_t)3 * 224 * 224 * 4, ob = (size_t)32 * d_.n_embd_llm * 4;
    memcpy(h_img_, image_host, ib);
    CUDA_CHECK(cudaMemcpyAsync(img_, h_img_, ib, cudaMemcpyHostToDevice, stream_));
    CUDA_CHECK(cudaEventRecord(ev0_, stream_));
    CUDA_CHECK(cudaGraphLaunch(graph_, stream_));
    CUDA_CHECK(cudaEventRecord(ev1_, stream_));
    CUDA_CHECK(cudaMemcpyAsync(h_out_, proj_out_, ob, cudaMemcpyDeviceToHost, stream_));
    launches_ += (unsigned long long)graph_kernels_;
}
float VisionDevice::encode_end(float *out_host) {
    CUDA_CHECK(cudaStreamSynchronize(stream_));
    memcpy(out_host, h_out_, (size_t)32 * d_.n_embd_llm * 4);
    float ms = 0.f; CUDA_CHECK(cudaEventElapsedTime(&ms, ev0_, ev1_));
    return ms;
}
float VisionDevice::encode(const float *image_host, float *out_host) { encode_begin(image_host); return encode_end(out_host); }
void VisionDevice::encode_taps(const float *image_host, float *embed, float *vit_blocks, float *ln_vision, float *qformer, float *out) {
    memcpy(h_img_, image_host, (size_t)3 * 224 * 224 * 4);
    CUDA_CHECK(cudaMemcpyAsync(img_, h_img_, (size_t)3 * 224 * 224 * 4, cudaMemcpyHostToDevice, stream_));
    const Taps taps{embed, vit_blocks, ln_vision, qformer, out};
    record(&taps);
    CUDA_CHECK(cudaStreamSynchronize(stream_));
}

// ------------------------------------------------------------------------------------------------
// kernel-level test hooks
// ------------------------------------------------------------------------------------------------
// out: [ksplit][T + 1 + (epi == GE_PATCH)][M] elements (F16 for GE_GELU_F16, F32 otherwise), pre-filled by the caller and copied back whole:
// a GE_PATCH output goes to rows 1..T, the others to rows 0..T-1, and the row after the last one written is a guard row.  With ksplit > 1,
// a plan that splits K (tsplit on, T > 128) writes its GE_PARTIAL slices to the grid.z leading slices; otherwise slice 0 is the output.
// aux: resid [T][M] (GE_RESID unless in_place, where the pre-filled rows of `out` are the residual) or pos [T + 1][M] (GE_PATCH).
int VisionDevice::test_gemm(int M, int T, int K, const void *w_f16, const void *x_f16, const float *bias, int epi, const float *aux, float qscale,
                            int qscale_rows, int ksplit, int tsplit, int in_place, void *out, int *plan_out) {
    const bool patch = epi == GE_PATCH, resid = epi == GE_RESID, gelu = epi == GE_GELU_F16;
    if (!gemm_shape_ok(M, K, T) || epi < GE_BIAS || epi > GE_PATCH || !w_f16 || !x_f16 || !out) return ErrFailedToAddString;
    if (ksplit < 1 || ksplit > 4 || (ksplit > 1 && !resid) || (in_place && !resid) || (!in_place && (resid || patch) && !aux)) return ErrFailedToAddString;
    const size_t R = (size_t)T + 1 + (patch ? 1 : 0), esz = gelu ? 2 : 4, obytes = (size_t)ksplit * R * M * esz;
    __half *W, *X, *tab = nullptr; float *B = nullptr, *A = nullptr; unsigned char *O;
    CUDA_CHECK(cudaMalloc((void **)&W, (size_t)M * K * 2)); CUDA_CHECK(cudaMalloc((void **)&X, (size_t)T * K * 2)); CUDA_CHECK(cudaMalloc((void **)&O, obytes));
    CUDA_CHECK(cudaMemcpy(W, w_f16, (size_t)M * K * 2, cudaMemcpyHostToDevice)); CUDA_CHECK(cudaMemcpy(X, x_f16, (size_t)T * K * 2, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(O, out, obytes, cudaMemcpyHostToDevice));
    if (bias) { CUDA_CHECK(cudaMalloc((void **)&B, (size_t)M * 4)); CUDA_CHECK(cudaMemcpy(B, bias, (size_t)M * 4, cudaMemcpyHostToDevice)); }
    if (aux && !in_place && (resid || patch)) {
        const size_t ab = (size_t)(patch ? T + 1 : T) * M * 4;
        CUDA_CHECK(cudaMalloc((void **)&A, ab)); CUDA_CHECK(cudaMemcpy(A, aux, ab, cudaMemcpyHostToDevice));
    }
    GemmPlan *p = make_plan(W, M, K, X, T, epi, tsplit != 0, ksplit);
    GemmArgs &g = p->a;
    g.bias = B; g.ld_out = M;
    if (gelu) { tab = upload_table(0); g.out_f16 = (__half *)O; g.tab_gelu = tab; }
    else g.out_f32 = (float *)O;
    if (epi == GE_QSCALE) { g.qscale = qscale; g.qscale_rows = qscale_rows; }
    if (resid) g.resid = in_place ? (const float *)O : A;
    if (patch) g.pos = A;
    if (g.epi == GE_PARTIAL) { g.partial = (float *)O; g.partial_stride = (long long)(R * M); }
    if (plan_out) { plan_out[0] = g.nt; plan_out[1] = p->grid_y; plan_out[2] = p->grid_z; plan_out[3] = g.k_split_blocks; }
    launch_plan(p, 0);
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(cudaMemcpy(out, O, obytes, cudaMemcpyDeviceToHost));
    delete p; cudaFree(W); cudaFree(X); cudaFree(O); if (B) cudaFree(B); if (A) cudaFree(A); if (tab) cudaFree(tab);
    return ErrNone;
}
int VisionDevice::test_dequant(int gg_type, const void *raw, long n, void *out_f16) {
    if (!vision_type_ok(gg_type) || n <= 0 || (gg_type != GG_F32 && gg_type != GG_F16 && n % 32)) return ErrLoadModelMiniGPT4DataType;
    HostTensor t; t.gg = gg_type; t.n_dims = 1; t.ne[0] = n; t.data = (const uint8_t *)raw;
    t.nbytes = (size_t)n / gg_block_elems(gg_type) * gg_block_bytes(gg_type);
    __half *d; CUDA_CHECK(cudaMalloc((void **)&d, (size_t)n * 2));
    put16(t, d);
    CUDA_CHECK(cudaMemcpy(out_f16, d, (size_t)n * 2, cudaMemcpyDeviceToHost));
    cudaFree(d);
    return ErrNone;
}
static void h16_to_host(void *dst, const __half *src, size_t n) { CUDA_CHECK(cudaMemcpy(dst, src, n * 2, cudaMemcpyDeviceToHost)); }
// layernorm_kernel as load() launches it: 128 threads per row, F16 and / or F32 outputs (the Q-Former's LayerNorms write both)
int VisionDevice::test_layernorm(const float *x, int rows, int n, const float *w, const float *b, float *out32, void *out16) {
    if (!x || !w || (!out32 && !out16) || rows < 1 || n < 1 || n > 1536) return ErrFailedToAddString;
    float *X, *W, *B = nullptr, *O = nullptr; __half *O16 = nullptr;
    const size_t N = (size_t)rows * n;
    CUDA_CHECK(cudaMalloc((void **)&X, N * 4)); CUDA_CHECK(cudaMalloc((void **)&W, (size_t)n * 4));
    CUDA_CHECK(cudaMemcpy(X, x, N * 4, cudaMemcpyHostToDevice)); CUDA_CHECK(cudaMemcpy(W, w, (size_t)n * 4, cudaMemcpyHostToDevice));
    if (b) { CUDA_CHECK(cudaMalloc((void **)&B, (size_t)n * 4)); CUDA_CHECK(cudaMemcpy(B, b, (size_t)n * 4, cudaMemcpyHostToDevice)); }
    if (out32) CUDA_CHECK(cudaMalloc((void **)&O, N * 4));
    if (out16) CUDA_CHECK(cudaMalloc((void **)&O16, N * 2));
    layernorm_kernel<<<rows, 128>>>(X, rows, n, W, B, O16, O, nullptr);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaDeviceSynchronize());
    if (out32) CUDA_CHECK(cudaMemcpy(out32, O, N * 4, cudaMemcpyDeviceToHost));
    if (out16) h16_to_host(out16, O16, N);
    cudaFree(X); cudaFree(W); if (B) cudaFree(B); if (O) cudaFree(O); if (O16) cudaFree(O16);
    return ErrNone;
}
// layernorm_fold_kernel: x (in / out) += parts[0] + ... + parts[n_parts - 1] in slice order (slice p at p * part_stride), then the F16 LayerNorm
int VisionDevice::test_layernorm_fold(float *x, int rows, int n, const float *w, const float *b, const float *parts, int n_parts, long long part_stride,
                                      void *out16) {
    if (!x || !w || !parts || !out16 || rows < 1 || n < 1 || n > 1536 || n_parts < 1 || part_stride < (long long)rows * n) return ErrFailedToAddString;
    const size_t N = (size_t)rows * n, P = (size_t)(n_parts - 1) * (size_t)part_stride + N;
    float *X, *W, *B = nullptr, *Pp; __half *O16;
    CUDA_CHECK(cudaMalloc((void **)&X, N * 4)); CUDA_CHECK(cudaMalloc((void **)&W, (size_t)n * 4)); CUDA_CHECK(cudaMalloc((void **)&Pp, P * 4));
    CUDA_CHECK(cudaMalloc((void **)&O16, N * 2));
    CUDA_CHECK(cudaMemcpy(X, x, N * 4, cudaMemcpyHostToDevice)); CUDA_CHECK(cudaMemcpy(W, w, (size_t)n * 4, cudaMemcpyHostToDevice));
    CUDA_CHECK(cudaMemcpy(Pp, parts, P * 4, cudaMemcpyHostToDevice));
    if (b) { CUDA_CHECK(cudaMalloc((void **)&B, (size_t)n * 4)); CUDA_CHECK(cudaMemcpy(B, b, (size_t)n * 4, cudaMemcpyHostToDevice)); }
    layernorm_fold_kernel<<<rows, 128>>>(X, rows, n, W, B, O16, Pp, n_parts, part_stride);
    CUDA_CHECK(cudaGetLastError());
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(cudaMemcpy(x, X, N * 4, cudaMemcpyDeviceToHost));
    h16_to_host(out16, O16, N);
    cudaFree(X); cudaFree(W); cudaFree(Pp); cudaFree(O16); if (B) cudaFree(B);
    return ErrNone;
}
// attention_f32_kernel as record() launches it: q / k / v at element offsets of one buffer (the packed qkv GEMM outputs), grid (heads,
// ceil(nq / q_per_cta)); q_per_cta 0: ceil(nq / 4).  out: [nq + 1][ld_out] F32, pre-filled by the caller; the kernel writes F16 values to
// columns < heads * dh of rows < nq, and the buffer comes back whole (row nq is a guard row).
int VisionDevice::test_attention(const float *buf, long long n_buf, long long q_off, int ldq, long long k_off, long long v_off, int ldkv, int nq, int nk,
                                 int heads, int dh, float div, int q_per_cta, int ld_out, float *out) {
    const long long w = (long long)heads * dh;
    auto span_ok = [&](long long off, int ld, int rows) { return off >= 0 && off % 4 == 0 && off + (long long)(rows - 1) * ld + w <= n_buf; };
    if (!buf || !out || (dh != 64 && dh != 88) || heads < 1 || nq < 1 || nk < 1 || nk > 288 || q_per_cta < 0) return ErrFailedToAddString;
    if (ldq < w || ldkv < w || ld_out < w || ldq % 4 || ldkv % 4 || !span_ok(q_off, ldq, nq) || !span_ok(k_off, ldkv, nk) || !span_ok(v_off, ldkv, nk))
        return ErrFailedToAddString;
    if (attn_smem(nk, dh) > (size_t)225 * 1024) return ErrFailedToAddString;   // (head_dim 88 fits at most 268 keys)
    const int qpc = q_per_cta ? q_per_cta : (nq + 3) / 4;
    const size_t ob = (size_t)(nq + 1) * ld_out;
    float *Bd; __half *O, *tab = upload_table(1);
    CUDA_CHECK(cudaMalloc((void **)&Bd, (size_t)n_buf * 4)); CUDA_CHECK(cudaMalloc((void **)&O, ob * 2));
    CUDA_CHECK(cudaMemcpy(Bd, buf, (size_t)n_buf * 4, cudaMemcpyHostToDevice));
    std::vector<__half> h(ob);
    for (size_t i = 0; i < ob; ++i) h[i] = __float2half_rn(out[i]);
    CUDA_CHECK(cudaMemcpy(O, h.data(), ob * 2, cudaMemcpyHostToDevice));
    launch_attention(dh, dim3((unsigned)heads, (unsigned)((nq + qpc - 1) / qpc)), 0, Bd + q_off, ldq, Bd + k_off, Bd + v_off, ldkv, nq, nk, div, qpc, O, ld_out, tab);
    CUDA_CHECK(cudaDeviceSynchronize());
    CUDA_CHECK(cudaMemcpy(h.data(), O, ob * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < ob; ++i) out[i] = __half2float(h[i]);
    cudaFree(Bd); cudaFree(O); cudaFree(tab);
    return ErrNone;
}

}  // namespace mg4

// vision.h — device-resident vision graph: EVA ViT-g/14 -> ln_vision -> Q-Former -> llama_proj
// (reference MiniGPT4::encode_image, minigpt4.cpp:2094-2363, and the layer functors :1014-1463).
//
// HBM layout: every >=2-D "*weight" tensor stays F16 row-major [out][in] (the container's own layout, ggml
// ne=[in,out]) and is consumed in place by TMA; the patch-embed kernel is re-laid to [1408][640] (K 588 padded
// to a multiple of 64); q_bias|0|v_bias are concatenated into one 4224-vector; Q-Former q/k/v (self) and k/v
// (cross) weights are concatenated so each attention needs one or two GEMMs.  Activations: F32 residual stream
// [257][1408], F16 GEMM operands.  The whole encode is one CUDA graph (static shapes).
#pragma once
#include "formats.h"
#include <cuda.h>
#include <functional>
#include <map>
#include <memory>

namespace mg4 {

struct VisionDims { int D = 1408, T = 257, H = 16, dh = 88, FF = 6144, n_blocks = 0, n_q = 32, qh = 768, q_layers = 0, n_embd_llm = 4096; };

struct GemmPlan;  // one planned wgmma GEMM launch (tensor maps + args)

class VisionDevice {
public:
    VisionDevice();
    ~VisionDevice();
    // share != null: a further LANE of the same model (batched encoding): weights are shared with `share`, activations / plans / graph / stream are this lane's own
    Error load(const VisionFile &f, const VisionDevice *share = nullptr);
    const VisionDims &dims() const { return d_; }
    // image: host F32 CHW [3][224][224]; out: host F32 [32][n_embd_llm].  Synchronous.  Returns device ms of the graph.
    float encode(const float *image_host, float *out_host);
    void encode_begin(const float *image_host);   // asynchronous half of encode() (several lanes run concurrently) ...
    float encode_end(float *out_host);            // ... and its synchronising half
    const float *last_embedding_device() const { return proj_out_; }
    // The forward of encode(), run eagerly on this lane's stream (not the graph) with every stage copied to the host as it becomes complete.
    // Each pointer may be null.  embed [T][D]: patch embedding + CLS + pos; vit_blocks [n_blocks][T][D]: the residual stream after each block;
    // ln_vision [T][D]: the F16 Q-Former operand as F32; qformer [q_layers][32][768]: hs after each layer; out [32][n_embd_llm].
    void encode_taps(const float *image_host, float *embed, float *vit_blocks, float *ln_vision, float *qformer, float *out);
    unsigned long long kernel_launches() const { return launches_; }
    double flops_per_image() const { return flops_; }
    size_t weight_bytes() const { return weight_bytes_; }
    cudaStream_t stream() const { return stream_; }

    // Kernel-level test seams: each runs one production kernel with the launch configuration load() / record() would give it and returns
    // ErrFailedToAddString (8) for arguments the kernel cannot take, before any device work.
    // out[T][M] = epi(W[M][K] . X[T][K]^T) through the wgmma GEMM; `out` is the caller's pre-filled buffer with one guard row past the last row
    // written (see minigpt4_b200_op_gemm_f16); plan_out (may be null) = {token tile, grid.y, grid.z, k-blocks per slice}.
    static int test_gemm(int M, int T, int K, const void *w_f16, const void *x_f16, const float *bias, int epi, const float *aux, float qscale,
                         int qscale_rows, int ksplit, int tsplit, int in_place, void *out, int *plan_out);
    static int test_dequant(int gg_type, const void *raw, long n, void *out_f16);
    static int test_layernorm(const float *x, int rows, int n, const float *w, const float *b, float *out32, void *out16);
    static int test_layernorm_fold(float *x, int rows, int n, const float *w, const float *b, const float *parts, int n_parts, long long part_stride,
                                   void *out16);
    static int test_attention(const float *buf, long long n_buf, long long q_off, int ldq, long long k_off, long long v_off, int ldkv, int nq, int nk,
                              int heads, int dh, float div, int q_per_cta, int ld_out, float *out);

private:
    struct Taps { float *embed, *vit_blocks, *ln_vision, *qformer, *out; };
    void record(const Taps *taps = nullptr);  // enqueue the whole forward on stream_ (captured into graph_ without taps)
    VisionDims d_;
    std::vector<GemmPlan *> plans_;
    std::vector<void *> allocs_;
    void *dalloc(size_t n);
    std::shared_ptr<std::map<std::string, void *>> wcache_;   // key -> device pointer of a weight (owned by the lane that uploaded it)
    void *cached(const std::string &key, size_t bytes, const std::function<void(void *)> &fill);
    static void put16(const HostTensor &t, __half *dst);  // any supported matrix type -> F16 on the device
    const __half *w16(const VisionFile &f, const std::string &model, const std::string &name, int rows, int cols);
    const float *w32(const VisionFile &f, const std::string &model, const std::string &name, int n);
    // weights
    struct Block { const float *n1w, *n1b, *n2w, *n2b, *qkv_bias, *proj_b, *fc1_b, *fc2_b; GemmPlan *qkv, *proj, *fc1, *fc2; };
    struct QLayer {
        const float *sa_qkv_b, *sa_o_b, *sa_ln_w, *sa_ln_b; GemmPlan *sa_qkv, *sa_o;
        bool cross = false; const float *ca_q_b, *ca_kv_b, *ca_o_b, *ca_ln_w, *ca_ln_b; GemmPlan *ca_q = nullptr, *ca_kv = nullptr, *ca_o = nullptr;
        const float *ff1_b, *ff2_b, *ff_ln_w, *ff_ln_b; GemmPlan *ff1, *ff2;
    };
    std::vector<Block> blocks_;
    std::vector<QLayer> qlayers_;
    GemmPlan *patch_ = nullptr, *proj_ = nullptr;
    const float *cls_ = nullptr, *pos_ = nullptr, *lnv_w_ = nullptr, *lnv_b_ = nullptr, *qtok_ = nullptr, *qln_w_ = nullptr, *qln_b_ = nullptr;
    // activations
    float *img_ = nullptr, *x_ = nullptr, *qkv_ = nullptr, *proj_out_ = nullptr;
    int splitk_ = 1; float *parts_ = nullptr;  // split-K slices of the residual GEMMs proj / fc2 (default 3)
    __half *patches_ = nullptr, *ln16_ = nullptr, *ctx16_ = nullptr, *h16_ = nullptr, *img_emb16_ = nullptr;
    float *qtmp_ = nullptr;
    float *hs_ = nullptr, *qa_ = nullptr, *qc_ = nullptr, *qqkv_ = nullptr, *qq_ = nullptr, *qkv_cross_ = nullptr;
    __half *hs16_ = nullptr, *qa16_ = nullptr, *qc16_ = nullptr, *qctx16_ = nullptr, *qh16_ = nullptr;
    __half *tab_gelu_ = nullptr, *tab_exp_ = nullptr;
    float *h_out_ = nullptr;  // pinned
    float *h_img_ = nullptr;  // pinned
    cudaStream_t stream_ = nullptr;
    cudaGraphExec_t graph_ = nullptr;
    cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
    unsigned long long launches_ = 0; int graph_kernels_ = 0;
    double flops_ = 0; size_t weight_bytes_ = 0;
};

}  // namespace mg4

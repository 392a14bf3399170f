// common.h — shared host-side declarations of the H100-native engine.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string>
#include <vector>

namespace mg4 {

// Error ordinals are ABI: callers receive them as plain ints and map them back through
// minigpt4_error_code_to_string (reference minigpt4.cpp:97-119, same order).
enum Error : int {
    ErrNone = 0,
    ErrLoadModelFileHeader,
    ErrLoadModelFileVersion,
    ErrLoadModelMiniGPT4DataType,
    ErrLoadLanguageModel,
    ErrOpenImage,
    ErrImageSize,
    ErrMmapSupport,
    ErrFailedToAddString,
    ErrLLamaProjectionEmbeddingInvalidSize,
    ErrFailedToAddEmbedding,
    ErrEosToken,
    ErrEos,
    ErrImageNot224_244_3,
    ErrImageNotF32,
    ErrImageChannelsExpectedRGB,
    ErrImageFormatExpectedU8,
    ErrPathDoesNotExist,
    ErrDumpModelFileOpen,
    ErrOpenCVNotLinked,
    ErrCount
};
const char *error_name(int code);

// process-global verbosity, like the reference's global_verbosity (minigpt4.cpp:152)
extern int g_verbosity;  // 0 none, 1 error, 2 info, 3 debug
#define MG4_ERR(...)  do { if (mg4::g_verbosity >= 1) { fprintf(stderr, "[minigpt4-b200][error] " __VA_ARGS__); fputc('\n', stderr); } } while (0)
#define MG4_INFO(...) do { if (mg4::g_verbosity >= 2) { fprintf(stdout, "[minigpt4-b200][info] " __VA_ARGS__); fputc('\n', stdout); } } while (0)
#define MG4_DBG(...)  do { if (mg4::g_verbosity >= 3) { fprintf(stdout, "[minigpt4-b200][debug] " __VA_ARGS__); fputc('\n', stdout); } } while (0)

// There is NO CPU fallback, so a failure is either reported or fatal - never worked around:
//  * while a model is being LOADED (a LoadScope is alive on this thread) a failed check - missing tensor, unsupported tensor type or shape,
//    device memory exhausted, no usable driver - throws LoadFailure; Engine::init turns it into the ABI's error code and
//    minigpt4_model_load returns NULL, like the reference (minigpt4.cpp:2476-2492);
//  * anywhere else (a kernel launch that failed, a corrupted context) the process aborts loudly (reference PANIC -> exit(-1), minigpt4.cpp:230-232).
struct LoadFailure { char msg[384]; };
extern thread_local int g_load_depth;
struct LoadScope { LoadScope() { ++g_load_depth; } ~LoadScope() { --g_load_depth; } };
[[noreturn]] void fail(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
[[noreturn]] void fail_cuda(cudaError_t e, const char *file, int line);
#define CUDA_CHECK(expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) mg4::fail_cuda(_e, __FILE__, __LINE__); } while (0)
#define MG4_PANIC(...) mg4::fail(__VA_ARGS__)

// ggml tensor type ids as stored in ggjt files (llama.cpp@master-31cfbb1 ggml.h)
enum GGType : int { GG_F32 = 0, GG_F16 = 1, GG_Q4_0 = 2, GG_Q4_1 = 3, GG_Q5_0 = 6, GG_Q5_1 = 7, GG_Q8_0 = 8, GG_Q8_1 = 9,
                    GG_Q2_K = 10, GG_Q3_K = 11, GG_Q4_K = 12, GG_Q5_K = 13, GG_Q6_K = 14, GG_Q8_K = 15, GG_I32 = 18, GG_COUNT = 19 };

// container dtype ids (include/minigpt4.h MiniGPT4DataType; mapping = reference minigpt4.cpp:555-739)
int container_dtype_to_gg(int dt);   // -1 if unknown
int gg_to_container_dtype(int gg);
size_t gg_block_elems(int gg);       // elements per block
size_t gg_block_bytes(int gg);       // bytes per block
inline size_t gg_row_bytes(int gg, size_t cols) { return cols / gg_block_elems(gg) * gg_block_bytes(gg); }

struct HostTensor {
    std::string name;
    int gg = -1;
    int n_dims = 0;
    int64_t ne[4] = {1, 1, 1, 1};
    const uint8_t *data = nullptr;  // view into the mapped file
    size_t nbytes = 0;
    int64_t nelements() const { return ne[0] * ne[1] * ne[2] * ne[3]; }
};

double now_ms();

// Sampler::sample's arguments, on the host (text.h) and the device (llama_sample.cuh): the non-mirostat chain (mirostat 0), or mirostat
// 1 / 2, which ignores top_k .. typical_p
struct SamplingArgs { float temp; int32_t top_k; float top_p, tfs_z, typical_p; int mirostat; float mirostat_tau, mirostat_eta; };
// the arguments of a call with these settings: with mirostat 1 / 2 top_k .. typical_p are neutral, with the chain tau and eta are 0
inline SamplingArgs sampling_args(float temp, int32_t top_k, float top_p, float tfs_z, float typical_p, int mirostat, float mirostat_tau,
                                  float mirostat_eta) {
    return mirostat ? SamplingArgs{temp, 0, 1.f, 1.f, 1.f, mirostat, mirostat_tau, mirostat_eta} : SamplingArgs{temp, top_k, top_p, tfs_z, typical_p};
}

}  // namespace mg4

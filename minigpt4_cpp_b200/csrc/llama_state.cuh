// llama_state.cuh — sm_90a kernel of minigpt4_b200_session_copy (host side LlamaDevice::copy_state in llama.cu, DESIGN.md §4.11).
//
// A conversation is its K / V rows 0 .. n_past - 1, its logits and its DeviceState: the attention kernels never read a key above a row's
// position, so rows >= n_past need no copy.  The KV layout is F16 [layer][n_ctx][n_embd], so each of the 2 n_layer planes contributes one
// contiguous run of n_past * n_embd halves (a multiple of 16 bytes: n_embd is a multiple of 128).  One launch fans the source out to
// every destination: each 16-byte chunk of the source is loaded once and stored to all n destinations at the same offset.
#pragma once
#include <cuda_runtime.h>
#include "llama.h"

namespace mg4 {
namespace k {

constexpr int kCopyMax = 64;        // LlamaDevice::kMaxBatch
constexpr int kCopyThreads = 256;
constexpr int kCopyUnroll = 4;      // chunks in flight per thread

// destinations travel in the parameter list (64 x 4 pointers = 2 KiB): no device table, no upload before the launch
struct CopyStateArgs {
    const uint4 *k, *v;             // source caches (layer 0)
    const float *logits;
    const DeviceState *state;
    uint4 *dk[kCopyMax], *dv[kCopyMax];
    float *dlogits[kCopyMax];
    DeviceState *dstate[kCopyMax];
    long long plane;                // 16-byte chunks of one layer's cache: n_ctx * n_embd * 2 / 16
    long long run;                  // 16-byte chunks copied of each plane: n_past * n_embd * 2 / 16
    int n;                          // destinations
    int n_layer, n_vocab;
};

// grid (x, 2 n_layer + 1), block kCopyThreads.  Row y < n_layer: K plane y; y < 2 n_layer: V plane y - n_layer; the last row: the logits
// (floats: n_vocab need not be a multiple of 4) and the 64-byte DeviceState.  Within a row the x blocks stride over the run, each thread
// keeping kCopyUnroll loads in flight before it stores them.
__global__ void __launch_bounds__(kCopyThreads) copy_state_kernel(const __grid_constant__ CopyStateArgs a) {
    const int y = (int)blockIdx.y;
    const long long stride = (long long)gridDim.x * kCopyThreads;
    const long long t0 = (long long)blockIdx.x * kCopyThreads + threadIdx.x;
    if (y < 2 * a.n_layer) {
        const bool is_v = y >= a.n_layer;
        const long long base = (long long)(is_v ? y - a.n_layer : y) * a.plane;
        const uint4 *__restrict__ src = (is_v ? a.v : a.k) + base;
        for (long long i0 = t0; i0 < a.run; i0 += stride * kCopyUnroll) {
            uint4 val[kCopyUnroll];
#pragma unroll
            for (int u = 0; u < kCopyUnroll; ++u) {
                const long long i = i0 + u * stride;
                if (i < a.run) val[u] = src[i];
            }
            for (int d = 0; d < a.n; ++d) {
                uint4 *__restrict__ dst = (is_v ? a.dv[d] : a.dk[d]) + base;
#pragma unroll
                for (int u = 0; u < kCopyUnroll; ++u) {
                    const long long i = i0 + u * stride;
                    if (i < a.run) dst[i] = val[u];
                }
            }
        }
        return;
    }
    for (long long i = t0; i < a.n_vocab; i += stride) {
        const float z = a.logits[i];
        for (int d = 0; d < a.n; ++d) a.dlogits[d][i] = z;
    }
    if (blockIdx.x == 0 && threadIdx.x < sizeof(DeviceState) / 4) {
        const int w = ((const int *)a.state)[threadIdx.x];
        for (int d = 0; d < a.n; ++d) ((int *)a.dstate[d])[threadIdx.x] = w;
    }
}

}  // namespace k
}  // namespace mg4

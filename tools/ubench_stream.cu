// ubench_stream.cu — primitive measurements behind the decode megakernel design (stand-alone; nvcc -arch=sm_90a).
//   T1  per-warp self-refilled TMA stream: every consumer warp owns two shared-memory slots and re-arms a slot itself right after
//       consuming it (no producer warp, no "empty" barriers).  work = 0 (wait only), 1 (read the slot), 2 (Q4_1 dot, register activations)
//   T2  T1 + a warp that asks L2 for the CTA's stream `window` bytes ahead (cp.async.bulk.prefetch.L2)
//   T4  grid barrier round trip, variants
//   T5  grid barrier + every CTA gathers a 16 KB vector from L2 (the activation exchange of one op)
//   T6  direct global->register streaming (ld.global.nc.v4, 8 in flight per lane)
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o build/ubench_stream tools/ubench_stream.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cuda_runtime.h>
#include <cooperative_groups.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count)); }
__device__ __forceinline__ void mb_expect_tx(uint64_t *bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mb_wait(uint64_t *bar, uint32_t parity) {
    asm volatile("{\n\t.reg .pred p;\n\tW:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D;\n\tbra W;\n\tD:\n\t}" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c) { int d; asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int q4_block_idot(const uint4 q, const int4 lo, const int4 hi) {
    int sl = dp4a_us(q.x & 0x0F0F0F0Fu, lo.x, 0), sh = dp4a_us(q.x & 0xF0F0F0F0u, hi.x, 0);
    sl = dp4a_us(q.y & 0x0F0F0F0Fu, lo.y, sl); sh = dp4a_us(q.y & 0xF0F0F0F0u, hi.y, sh);
    sl = dp4a_us(q.z & 0x0F0F0F0Fu, lo.z, sl); sh = dp4a_us(q.z & 0xF0F0F0F0u, hi.z, sh);
    sl = dp4a_us(q.w & 0x0F0F0F0Fu, lo.w, sl); sh = dp4a_us(q.w & 0xF0F0F0F0u, hi.w, sh);
    return sl + (sh >> 4);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

constexpr int kSlot = 6912;  // >= one 11008-wide Q4_1 row (6880 B), 128-byte multiple
constexpr int kW = 15;

// T1 / T2
template <int WORK>
__global__ void __launch_bounds__(512, 1) stream_kernel(const unsigned char *__restrict__ w, size_t per_cta, int load_bytes, int window, float *sink, unsigned long long *clk) {
    extern __shared__ __align__(128) unsigned char smem[];
    uint64_t *full = (uint64_t *)(smem + (size_t)2 * kW * kSlot);
    volatile unsigned *filled = (volatile unsigned *)(full + 2 * kW);  // slot-loads issued so far by the consumers of this CTA
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) { for (int s = 0; s < 2 * kW; ++s) mb_init(&full[s], 1); *filled = 2 * kW; asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    const unsigned char *base = w + (size_t)blockIdx.x * per_cta;
    const int n_loads = (int)(per_cta / (size_t)load_bytes);
    long long t0 = clock64();
    if (warp == kW) {
        if (window > 0 && lane == 0) {
            const int ahead = window / load_bytes;
            for (int i = 2 * kW; i < n_loads; ++i) {
                while (i - (int)*filled > ahead) __nanosleep(64);
                if (i > (int)*filled) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(base + (size_t)i * load_bytes), "r"(load_bytes) : "memory");
            }
        }
        return;
    }
    unsigned char *slot[2] = {smem + (size_t)(2 * warp) * kSlot, smem + (size_t)(2 * warp + 1) * kSlot};
    uint64_t *fb[2] = {&full[2 * warp], &full[2 * warp + 1]};
    int nf = warp;  // next slot-load to request
    if (lane == 0) {
        for (int j = 0; j < 2; ++j) if (nf < n_loads) { mb_expect_tx(fb[j], load_bytes); bulk_g2s(slot[j], base + (size_t)nf * load_bytes, load_bytes, fb[j]); nf += kW; }
    }
    nf = warp + 2 * kW;
    int4 alo[4], ahi[4]; float ad[4], as[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { alo[i] = make_int4(lane + i, lane * 3, i, 7); ahi[i] = make_int4(lane, i, 5, lane + 9); ad[i] = 0.01f * (lane + 1); as[i] = 0.5f; }
    float acc = 0.f; unsigned x = 0;
    int it = 0;
    for (int n = warp; n < n_loads; n += kW, ++it) {
        const int j = it & 1; const unsigned ph = (it >> 1) & 1;
        mb_wait(fb[j], ph);
        const unsigned char *s = slot[j];
        if (WORK == 1) {
            for (int o = lane * 16; o < load_bytes; o += 512) { const uint4 v = *(const uint4 *)(s + o); x ^= v.x ^ v.y ^ v.z ^ v.w; }
        } else if (WORK == 2) {
            // two Q4_1 rows of 4096 columns: [128 x 16 B nibbles][128 x half2] per row (2560 B); register-resident activations
            const uint4 *q0p = (const uint4 *)s, *q1p = (const uint4 *)(s + 2560);
            const __half2 *s0p = (const __half2 *)(s + 2048), *s1p = (const __half2 *)(s + 2560 + 2048);
            float d0 = 0.f, m0 = 0.f, d1 = 0.f, m1 = 0.f;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int b = lane + 32 * i;
                const uint4 q0 = q0p[b], q1 = q1p[b];
                const int i0 = q4_block_idot(q0, alo[i], ahi[i]), i1 = q4_block_idot(q1, alo[i], ahi[i]);
                const float2 f0 = __half22float2(s0p[b]), f1 = __half22float2(s1p[b]);
                d0 = fmaf(f0.x * ad[i], (float)i0, d0); m0 = fmaf(f0.y, as[i], m0);
                d1 = fmaf(f1.x * ad[i], (float)i1, d1); m1 = fmaf(f1.y, as[i], m1);
            }
            __syncwarp();
            if (lane == 0 && nf < n_loads) { mb_expect_tx(fb[j], load_bytes); bulk_g2s(slot[j], base + (size_t)nf * load_bytes, load_bytes, fb[j]); atomicAdd((unsigned *)filled, 1u); }
            nf += kW;
            acc += (warp_sum(d0) + warp_sum(m0)) + (warp_sum(d1) + warp_sum(m1));
            continue;
        }
        __syncwarp();
        if (lane == 0 && nf < n_loads) { mb_expect_tx(fb[j], load_bytes); bulk_g2s(slot[j], base + (size_t)nf * load_bytes, load_bytes, fb[j]); atomicAdd((unsigned *)filled, 1u); }
        nf += kW;
    }
    if (acc == 123.456f || x == 0x12345u) sink[0] = acc + x;
    if (tid == 0 && clk) clk[blockIdx.x] = (unsigned long long)(clock64() - t0);
}

// T6: direct register streaming
__global__ void __launch_bounds__(512, 1) ldg_kernel(const uint4 *__restrict__ w, size_t per_cta16, float *sink) {
    const uint4 *base = w + (size_t)blockIdx.x * per_cta16;
    unsigned x = 0;
    for (size_t i = threadIdx.x; i + 7 * 512 < per_cta16; i += 8 * 512) {
        uint4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v[u].x), "=r"(v[u].y), "=r"(v[u].z), "=r"(v[u].w) : "l"(base + i + u * 512));
#pragma unroll
        for (int u = 0; u < 8; ++u) x ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
    }
    if (x == 0x12345u) sink[0] = x;
}

// T4 / T5: grid barrier variants
template <int VAR>
__device__ __forceinline__ void grid_barrier(unsigned *counter, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        if (VAR == 0) { asm volatile("fence.acq_rel.gpu;" ::: "memory"); asm volatile("red.relaxed.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory"); }
        else asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
        unsigned v;
        if (VAR == 2) { do { asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory"); } while (v < target); asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
        else do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory"); } while (v < target);
    }
    __syncthreads();
}
template <int VAR, bool GATHER>
__global__ void __launch_bounds__(512, 1) barrier_kernel(unsigned *counter, float *vec, int iters, float *sink) {
    __shared__ float red[16];
    float acc = 0.f;
    for (int i = 0; i < iters; ++i) {
        if (GATHER) {  // every CTA writes its 1/G of the 4096-vector, then everybody reads all of it (ld.global.cg)
            const int G = gridDim.x;
            for (int e = blockIdx.x * 4096 / G + threadIdx.x; e < (blockIdx.x + 1) * 4096 / G; e += 512) vec[e] = (float)(i + e);
        }
        grid_barrier<VAR>(counter, (unsigned)(i + 1) * gridDim.x);
        if (GATHER) {
            if (threadIdx.x < 256) {
                float4 v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) v[u] = __ldcg((const float4 *)vec + threadIdx.x + 256 * u);
                float s = 0.f;
#pragma unroll
                for (int u = 0; u < 4; ++u) s += v[u].x * v[u].x + v[u].y * v[u].y + v[u].z * v[u].z + v[u].w * v[u].w;
                s = warp_sum(s);
                if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
            }
            __syncthreads();
            acc += red[0] + red[1] + red[2] + red[3] + red[4] + red[5] + red[6] + red[7];
        }
    }
    if (acc == 123.f) sink[0] = acc;
}

template <typename F> float time_ms(F f, int reps = 3) {
    cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    float best = 1e30f;
    for (int r = 0; r < reps; ++r) { CK(cudaEventRecord(a)); f(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b)); float ms; CK(cudaEventElapsedTime(&ms, a, b)); if (ms < best) best = ms; }
    return best;
}

int main() {
    setvbuf(stdout, nullptr, _IOLBF, 0);
    int dev = 0; cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, dev));
    const int G = prop.multiProcessorCount;
    printf("device %s, %d SMs\n", prop.name, G);
    const size_t total = (size_t)3 << 30;  // 3 GiB >> L2
    unsigned char *w; CK(cudaMalloc(&w, total + (1 << 20))); CK(cudaMemset(w, 0x5a, total + (1 << 20)));
    float *sink; CK(cudaMalloc(&sink, 64));
    unsigned *counter; CK(cudaMalloc(&counter, 256));
    float *vec; CK(cudaMalloc(&vec, 4096 * 4));
    const size_t smem = (size_t)2 * kW * kSlot + 2 * kW * 8 + 64;
    CK(cudaFuncSetAttribute(stream_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(stream_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(stream_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int load_bytes : {5120, 6880}) {
        const size_t per_cta = (total / G) / ((size_t)load_bytes * 16) * ((size_t)load_bytes * 16);  // 16-byte aligned sources
        const double gb = (double)per_cta * G / 1e9;
        for (int window : {0, 131072, 262144}) {
            float ms0 = time_ms([&] { stream_kernel<0><<<G, 512, smem>>>(w, per_cta, load_bytes, window, sink, nullptr); });
            float ms1 = time_ms([&] { stream_kernel<1><<<G, 512, smem>>>(w, per_cta, load_bytes, window, sink, nullptr); });
            float ms2 = load_bytes == 5120 ? time_ms([&] { stream_kernel<2><<<G, 512, smem>>>(w, per_cta, load_bytes, window, sink, nullptr); }) : 0.f;
            CK(cudaGetLastError());
            printf("T1/T2 self-refill load=%d B window=%6d B/CTA: wait-only %7.1f GB/s | read %7.1f GB/s | q4_1 dot (reg acts) %7.1f GB/s\n", load_bytes, window, gb / ms0 * 1e3, gb / ms1 * 1e3, ms2 > 0 ? gb / ms2 * 1e3 : 0.0);
        }
    }
    {
        const size_t per16 = total / G / 16;
        float ms = time_ms([&] { ldg_kernel<<<G, 512>>>((const uint4 *)w, per16, sink); });
        printf("T6 ldg.nc.v4 x8 per lane, 512 thr/SM: %7.1f GB/s\n", (double)per16 * 16 * G / 1e9 / ms * 1e3);
        float ms2 = time_ms([&] { ldg_kernel<<<2 * G, 512>>>((const uint4 *)w, per16 / 2, sink); });
        printf("T6 ldg.nc.v4 x8 per lane, 2 x 512 thr/SM: %7.1f GB/s\n", (double)(per16 / 2) * 16 * 2 * G / 1e9 / ms2 * 1e3);
    }
    const int iters = 2000;
    auto run_bar = [&](auto kern, const char *name) {
        CK(cudaMemset(counter, 0, 256));
        void *args[] = {(void *)&counter, (void *)&vec, (void *)&iters, (void *)&sink};
        cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
        CK(cudaEventRecord(a));
        CK(cudaLaunchCooperativeKernel((const void *)kern, dim3(G), dim3(512), args, 0, 0));
        CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
        float ms; CK(cudaEventElapsedTime(&ms, a, b));
        printf("%s: %.3f us per iteration\n", name, ms * 1e3 / iters);
    };
    run_bar(barrier_kernel<0, false>, "T4 barrier fence.acq_rel + red.relaxed + ld.acquire poll");
    run_bar(barrier_kernel<1, false>, "T4 barrier red.release + ld.acquire poll");
    run_bar(barrier_kernel<2, false>, "T4 barrier red.release + ld.relaxed poll + fence");
    run_bar(barrier_kernel<0, true>, "T5 write 1/G + barrier(v0) + gather 16 KB + sum");
    run_bar(barrier_kernel<1, true>, "T5 write 1/G + barrier(v1) + gather 16 KB + sum");
    run_bar(barrier_kernel<2, true>, "T5 write 1/G + barrier(v2) + gather 16 KB + sum");
    CK(cudaDeviceSynchronize());
    printf("done\n");
    return 0;
}

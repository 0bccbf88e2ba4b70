// Micro-benchmarks that size the streaming kernels of allegro_b200 :
//   bulk   : persistent CTAs, ONE producer thread issuing cp.async.bulk (global -> shared, mbarrier complete_tx)
//            into a ring of NS stages of CH bytes; NC consumer warps read every byte from shared memory.
//            -> achievable HBM read rate of a "TMA-staged CSR row" pipeline vs stage size / depth / CTAs per SM.
//   ldg    : plain coalesced LDG.128 streaming with U independent loads in flight per thread.
//   ffma   : FFMA issue throughput per SM.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o tools/ubench/ubench tools/ubench/ubench.cu
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x)                                                                              \
    do {                                                                                   \
        cudaError_t e = (x);                                                               \
        if (e != cudaSuccess) {                                                            \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); \
            exit(1);                                                                       \
        }                                                                                  \
    } while (0)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "W_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra W_DONE;\n\t"
        "bra W_LOOP;\n\t"
        "W_DONE:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
                 "r"(bytes), "r"(bar)
                 : "memory");
}

template <int NS>
__global__ void __launch_bounds__(288) bulk_kernel(const float* __restrict__ src, int64_t n_chunks, int CH, int NC, float* out) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem);  // full[NS], empty[NS]
    uint8_t* ring = smem + 128;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NS; ++s) {
            mbar_init(smem_u32(bars + s), 1);
            mbar_init(smem_u32(bars + NS + s), NC);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == NC) {
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
                mbar_wait(smem_u32(bars + NS + stage), phase ^ 1);
                mbar_expect_tx(smem_u32(bars + stage), CH);
                bulk_g2s(smem_u32(ring + (size_t)stage * CH), reinterpret_cast<const uint8_t*>(src) + c * (int64_t)CH, CH,
                         smem_u32(bars + stage));
                if (++stage == NS) { stage = 0; phase ^= 1; }
            }
        }
    } else if (warp < NC) {
        int stage = 0;
        uint32_t phase = 0;
        float acc = 0.f;
        for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
            mbar_wait(smem_u32(bars + stage), phase);
            const float4* p = reinterpret_cast<const float4*>(ring + (size_t)stage * CH);
            const int n4 = CH / 16;
            for (int i = warp * 32 + lane; i < n4; i += NC * 32) {
                const float4 v = p[i];
                acc += v.x + v.y + v.z + v.w;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_u32(bars + NS + stage));
            if (++stage == NS) { stage = 0; phase ^= 1; }
        }
        if (acc == 123.456f) out[0] = acc;
    }
}

template <int U>
__global__ void __launch_bounds__(256) ldg_kernel(const float4* __restrict__ src, int64_t n4, float* out) {
    float acc = 0.f;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; i + (U - 1) * stride < n4; i += U * stride) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) v[u] = __ldg(src + i + u * stride);
#pragma unroll
        for (int u = 0; u < U; ++u) acc += v[u].x + v[u].y + v[u].z + v[u].w;
    }
    if (acc == 123.456f) out[0] = acc;
}

// dependent-chain-free FMA loops: 16 independent accumulators (8 pairs)
__global__ void __launch_bounds__(256) ffma_kernel(float* out, int iters, float a, float b) {
    float2 acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = make_float2(threadIdx.x + i, threadIdx.x - i);
    float2 m = make_float2(a, a * 1.0001f), c = make_float2(b, b * 0.999f);
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(acc[i].x) : "f"(m.x), "f"(c.x));
            asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(acc[i].y) : "f"(m.y), "f"(c.y));
        }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += acc[i].x + acc[i].y;
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

static float time_ms(cudaEvent_t a, cudaEvent_t b) {
    float ms;
    CK(cudaEventElapsedTime(&ms, a, b));
    return ms;
}

int main() {
    int nsm = 0;
    CK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0));
    const size_t bytes = (size_t)2 << 30;  // 2 GiB >> L2
    float* src;
    float* out;
    CK(cudaMalloc(&src, bytes));
    CK(cudaMalloc(&out, 1 << 22));
    CK(cudaMemset(src, 0, bytes));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    printf("SMs %d\n", nsm);
    // ---- plain LDG ----
    {
        const int64_t n4 = bytes / 16;
        auto run = [&](auto kern, int U, int cps) {
            for (int r = 0; r < 3; ++r) {
                CK(cudaEventRecord(e0));
                kern<<<nsm * cps, 256>>>((const float4*)src, n4, out);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
            }
            printf("ldg   U=%d ctas/SM=%d : %.0f GB/s\n", U, cps, bytes / time_ms(e0, e1) / 1e6);
        };
        run(ldg_kernel<4>, 4, 4);
        run(ldg_kernel<8>, 8, 4);
        run(ldg_kernel<8>, 8, 8);
        run(ldg_kernel<16>, 16, 4);
    }
    // ---- bulk-copy pipeline ----
    {
        auto run = [&](auto kern, int NS, int CH, int NC, int cps) {
            const size_t smem = 128 + (size_t)NS * CH;
            if (smem * cps > 227 * 1024) return;
            CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            const int64_t n_chunks = bytes / CH;
            for (int r = 0; r < 3; ++r) {
                CK(cudaEventRecord(e0));
                kern<<<nsm * cps, (NC + 1) * 32, smem>>>(src, n_chunks, CH, NC, out);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
            }
            CK(cudaGetLastError());
            printf("bulk  NS=%d CH=%5d NC=%d ctas/SM=%d in-flight/SM=%4d KB : %.0f GB/s\n", NS, CH, NC, cps, NS * CH * cps / 1024,
                   bytes / time_ms(e0, e1) / 1e6);
        };
        for (int cps : {1, 2, 4}) {
            for (int CH : {4096, 8192, 16384, 32768}) {
                run(bulk_kernel<2>, 2, CH, 4, cps);
                run(bulk_kernel<3>, 3, CH, 4, cps);
                run(bulk_kernel<4>, 4, CH, 4, cps);
                run(bulk_kernel<6>, 6, CH, 4, cps);
            }
        }
        run(bulk_kernel<4>, 4, 16384, 8, 1);
        run(bulk_kernel<4>, 4, 16384, 8, 2);
        run(bulk_kernel<4>, 4, 1536, 4, 4);   // one edge of the c2 backward per copy (1152 + 384 B): small-copy limit
        run(bulk_kernel<6>, 6, 1536, 4, 4);
        run(bulk_kernel<6>, 6, 1536, 4, 8);
    }
    // ---- FFMA ----
    {
        const int iters = 4096;
        for (int r = 0; r < 3; ++r) {
            CK(cudaEventRecord(e0));
            ffma_kernel<<<nsm * 8, 256>>>(out, iters, 1.0001f, 0.5f);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
        }
        const double fma = (double)nsm * 8 * 256 * iters * 16;
        printf("FFMA : %.1f TFMA/s (%.1f FMA/clk/SM at 1.98 GHz)\n", fma / time_ms(e0, e1) / 1e9, fma / time_ms(e0, e1) / 1e3 / nsm / 1.98e6);
    }
    return 0;
}

// wgmma (Hopper warpgroup tensor core) path of the fused linear layer -- same contract as linear.cu:
//
//   Out[M][N] (+)= epi( act([A_0 | A_1 | ...])[M][K] @ W[K][N] )
//
// M = number of edges (10^5..10^8), K <= 512, N <= 128 per launch (wider outputs run as column
// slices): a tall-skinny GEMM that is HBM-bound once the MACs run on tensor cores (12-25 KFLOP per
// ~0.5-1 KB row).  Structure (one persistent CTA per SM, 16 warps, warp-specialised, hand-written PTX):
//
//   warps 0-7  producers : coalesced global loads of the concatenated A row segments
//                          (8 rows x 128 B per warp instruction), optional SiLU, split of the fp32
//                          value into bf16 hi + bf16 lo, 16-byte st.shared into a ring of
//                          128-row x 32-k stages in the GMMA canonical K-major (no-swizzle,
//                          8x16B core matrix) layout; fence.proxy.async + mbarrier arrive.
//   warps 8-15 consumers : two warpgroups, one per 64-row half of the tile.  Each issues
//                          wgmma.mma_async m64nNk16 (N = Npad <= 128) from shared-memory descriptors
//                          into register accumulators; fp32 storage uses the 3-term split
//                          A_hi W_hi + A_lo W_hi + A_hi W_lo (~2^-16 relative, fp32 accumulate).
//                          A ring slot is released once the wgmma group that read it has retired.
//                          The epilogue runs from the accumulator registers: staged per warp through
//                          shared memory, silu' / accumulate, split into the output column segments,
//                          vectorised global stores.
//
// W (all of it: <= 128 KB as bf16 hi+lo) is staged once per CTA from a pre-packed image
// (ab2_linear_pack) and stays resident in shared memory.
#include <cuda.h>

#include <type_traits>

#include "common.cuh"
#include "radial_basis.cuh"

extern int g_ab2_opt_linear_tc;
extern int g_ab2_opt_linear_tma;
extern int g_ab2_opt_tc_debug;  // bit0: no epilogue global stores, bit1: no producer global loads, bit2: no MMA issue

namespace {

constexpr int BM = 128;       // rows per tile = 2 consumer warpgroups x wgmma M (64)
constexpr int KC = 32;        // k per ring stage
constexpr int NSTAGE = 4;        // max ring stages (run-time count p.nstage <= NSTAGE)
constexpr int RAW_STAGE = 256 * 4 * 16;  // bytes: 256 producer threads x 4 x 16-byte chunks (x2 with aux)
constexpr int EPI_LD = 40;       // floats per staged row (32 + 8 pad): conflict-free float2 writes / float4 reads
constexpr int NCONS = 8;         // consumer warps (2 warpgroups)
constexpr int EPI_BYTES = NCONS * 16 * EPI_LD * 4;  // 16 rows x 32 columns per consumer warp
constexpr int STAGE_HALF = BM * KC * 2;  // bytes of one bf16 [128][32] operand image (8 KB)
constexpr int NPROD = 8;                       // producer warps
constexpr int NTHREADS = (NPROD + NCONS) * 32;  // producers + consumers
constexpr int MAX_W_BYTES = 128 * 1024;
constexpr int MAX_K = 512;                     // k-chunk table size (MAX_K / 8 entries)
constexpr int MAX_N = 128;                     // columns per launch: wgmma N <= 128 keeps the accumulator at 64 registers
constexpr int MAX_CHUNK = MAX_N / 32;          // 32-column output chunks
// tail of the shared-memory plan: barriers | output chunk table | A / aux k-chunk tables
constexpr int TAIL_BARS = 2 * NSTAGE * 8, TAIL_CHUNK = MAX_CHUNK * 32, TAIL_KMAP = (MAX_K / 8) * 16;
constexpr int TAIL_BYTES = TAIL_BARS + TAIL_CHUNK + 2 * TAIL_KMAP;

struct TcSeg {
    const void* ptr;
    int64_t ld;
    int width;
    int accum;
    const void* aux;   // A segments: silu' multiplier source (AB2_ACT_MUL_DSILU), may be null
    int64_t aux_ld;
};

struct TcParams {
    int64_t M;
    int K, N, Npad;
    int n_a;
    TcSeg a[AB2_MAX_SEG];
    int act;
    const void* Wpacked;  // hi image of this column slice: Npad*K bf16 in canonical layout
    const void* Wlo;      // lo image of the same slice (fp32 storage only)
    int n_o;
    TcSeg o[AB2_MAX_SEG];
    int epi;
    const void* aux;
    int64_t aux_ld;
    int64_t num_tiles;
    int nstage;
    int debug;
    int raw_depth;  // cp.async stages in flight per producer thread (2 or 4)
    int has_aux;    // act == AB2_ACT_MUL_DSILU: the raw slots carry A and aux chunks
};

// Address tables built once per CTA so that the per-item / per-chunk code of the producer and
// epilogue warps is a shared-memory lookup plus 32-bit offsets.  (Walking the segment list and doing
// 64-bit index arithmetic per access makes both warp groups instruction-latency bound.)
struct KEnt {        // source of concat columns [8e, 8e+8): pointer to (row 0, that column), row stride
    const void* ptr; // null: beyond K (or, in the aux table, a segment without silu' multiplier)
    int64_t ld;      // elements
};
struct ChunkInfo {   // 32-column output chunk c0 = 32*i
    float* optr;       // (row 0, column c0) of the output segment that contains the chunk
    const float* aptr; // (row 0, column c0) of the silu' aux matrix
    int64_t ld;        // output row stride (elements)
    int32_t accum;
    int32_t ok;        // 1: chunk lies inside one fp32 segment, 16-byte aligned -> coalesced path
};
static_assert(sizeof(KEnt) == 16 && sizeof(ChunkInfo) == 32, "table entry sizes");

// ---- PTX wrappers ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// ---- wgmma (sm_90a) ----
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64][32*NCH] (+)= A[smem desc] * B[smem desc]^T, bf16 inputs, both K-major, fp32 accumulate in registers.
// Accumulator fragment of thread (warp w of the warpgroup, lane l): d[4j + {0,1}] = row 16w + l/4,
// columns 8j + 2(l%4) + {0,1}; d[4j + {2,3}] = the same columns of row 16w + l/4 + 8.
template <int NCH>
__device__ __forceinline__ void wgmma_bf16(float (&d)[16 * NCH], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (NCH == 1) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(da), "l"(db), "r"(scale_d));
    } else if constexpr (NCH == 2) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(da), "l"(db), "r"(scale_d));
    } else if constexpr (NCH == 3) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
            : "l"(da), "l"(db), "r"(scale_d));
    } else if constexpr (NCH == 4) {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
            : "l"(da), "l"(db), "r"(scale_d));
    }

}

__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst_smem, const void* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// explicit global-space accesses (table pointers come out of shared memory, so the compiler would
// otherwise emit generic LD/ST)
__device__ __forceinline__ void stg128(float* p, const float4& v) {
    asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 ldg128(const float* p) {
    float4 v;
    asm volatile("ld.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float4 ldg128_nc(const float* p) {
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

// global address of concat columns [k, k+8) of row m (nullptr if outside K)
template <typename TSrc>
__device__ __forceinline__ const TSrc* seg_ptr(const TcParams& p, int64_t m, int k) {
#pragma unroll
    for (int s = 0; s < AB2_MAX_SEG; ++s) {
        if (s < p.n_a) {
            if (k < p.a[s].width) return (const TSrc*)p.a[s].ptr + m * p.a[s].ld + k;
            k -= p.a[s].width;
        }
    }
    return nullptr;
}

template <typename TSrc>
__device__ __forceinline__ const TSrc* seg_aux_ptr(const TcParams& p, int64_t m, int k) {
#pragma unroll
    for (int s = 0; s < AB2_MAX_SEG; ++s) {
        if (s < p.n_a) {
            if (k < p.a[s].width) return p.a[s].aux ? (const TSrc*)p.a[s].aux + m * p.a[s].aux_ld + k : nullptr;
            k -= p.a[s].width;
        }
    }
    return nullptr;
}

// wgmma shared-memory matrix descriptor: K-major, no swizzle (interleave), 8x16B core matrices.
// canonical layout (16-byte units) ((8,n),2):((1,SBO),LBO): LBO = byte distance between core
// matrices adjacent in K, SBO = between 8-row groups.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;  // base_offset = 0, layout_type = 0 (no swizzle)
}

// branch-free SiLU and SiLU' (MUFU ex2 / rcp, ~2 ulp): IEEE division has a slow-path branch that
// serialises the unrolled epilogue / producer loops.
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float silu_fast(float x) { return x * sigmoid_fast(x); }
__device__ __forceinline__ float dsilu_fast(float x) {
    const float sg = sigmoid_fast(x);
    return sg * (1.f + x * (1.f - sg));
}
// mish and mish' in the same style (the forms of mish_f / dmish_f in common.cuh): n = e^min(x, 20) keeps every
// denominator below 2^60, far inside the range where __fdividef is exact to ~2 ulp.  Finite for every finite x.
__device__ __forceinline__ float mish_fast(float x) {
    const float n = __expf(fminf(x, 20.f)), nn = n * (n + 2.f);
    return x * __fdividef(nn, nn + 2.f);
}
__device__ __forceinline__ float dmish_fast(float x) {
    const float xc = fminf(x, 20.f), n = __expf(xc), nn = n * (n + 2.f), r = __fdividef(1.f, nn + 2.f);
    const float t = nn * r;
    return t + xc * (2.f * r * (1.f + t)) * __fdividef(n, 1.f + n);
}
// gelu and gelu' (exact erf form): erfcf(-x / sqrt2) does not cancel for x < -3 as 1 + erff(x / sqrt2) does; the Gaussian
// factor underflows to 0 (not NaN) for |x| beyond ~13
__device__ __forceinline__ float gelu_fast(float x) { return 0.5f * x * erfcf(-x * 0.70710678118654752f); }
__device__ __forceinline__ float dgelu_fast(float x) {
    return 0.5f * erfcf(-x * 0.70710678118654752f) + x * __expf(-0.5f * x * x) * 0.39894228040143268f;
}
// the MLP nonlinearity NL (AB2_NL_*) and its derivative; AB2_NL_SILU is silu_fast / dsilu_fast exactly
template <int NL>
__device__ __forceinline__ float act_fast(float x) {
    if constexpr (NL == AB2_NL_MISH) return mish_fast(x);
    else if constexpr (NL == AB2_NL_GELU) return gelu_fast(x);
    else return silu_fast(x);
}
template <int NL>
__device__ __forceinline__ float dact_fast(float x) {
    if constexpr (NL == AB2_NL_MISH) return dmish_fast(x);
    else if constexpr (NL == AB2_NL_GELU) return dgelu_fast(x);
    else return dsilu_fast(x);
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}

// load 8 consecutive concat columns [k, k+8) of row m (segment widths are multiples of 8)
template <typename TSrc>
__device__ __forceinline__ void load8(const TcParams& p, int64_t m, int k, float (&v)[8]) {
#pragma unroll
    for (int s = 0; s < AB2_MAX_SEG; ++s) {
        if (s < p.n_a) {
            if (k < p.a[s].width) {
                if constexpr (sizeof(TSrc) == 4) {
                    const float4* src = reinterpret_cast<const float4*>((const float*)p.a[s].ptr + m * p.a[s].ld + k);
                    const float4 x = __ldg(src), y = __ldg(src + 1);
                    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w; v[4] = y.x; v[5] = y.y; v[6] = y.z; v[7] = y.w;
                } else {
                    const uint4 x = __ldg(reinterpret_cast<const uint4*>((const bf16*)p.a[s].ptr + m * p.a[s].ld + k));
                    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&x);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float2 f = __bfloat1622float2(h[t]);
                        v[2 * t] = f.x; v[2 * t + 1] = f.y;
                    }
                }
                return;
            }
            k -= p.a[s].width;
        }
    }
#pragma unroll
    for (int t = 0; t < 8; ++t) v[t] = 0.f;
}


// output chunk table entry for columns [c0, c0 + 32)
template <typename TSrc>
__device__ __forceinline__ ChunkInfo tc_chunk_info(const TcParams& p, int c0) {
    ChunkInfo info{nullptr, nullptr, 0, 0, 0};
    if (sizeof(TSrc) == 4 && c0 + 32 <= p.N && !(p.debug & 64)) {
        int lo = 0, seg = -1, seg_lo = 0;
#pragma unroll
        for (int s2 = 0; s2 < AB2_MAX_SEG; ++s2) {
            if (s2 < p.n_o) {
                if (c0 >= lo && c0 + 32 <= lo + p.o[s2].width) { seg = s2; seg_lo = lo; }
                lo += p.o[s2].width;
            }
        }
        if (seg >= 0) {
            float* base = (float*)p.o[seg].ptr + (c0 - seg_lo);
            bool ok = !(reinterpret_cast<uintptr_t>(base) & 15) && !((p.o[seg].ld * 4) & 15);
            if (p.epi == AB2_EPI_MUL_DSILU &&
                ((reinterpret_cast<uintptr_t>((const float*)p.aux + c0) & 15) || ((p.aux_ld * 4) & 15))) ok = false;
            info.optr = base;
            info.aptr = (const float*)p.aux + c0;
            info.ld = p.o[seg].ld;
            info.accum = p.o[seg].accum;
            info.ok = ok ? 1 : 0;
        }
    }
    return info;
}

// Shared-memory / barrier context of one CTA, common to the cp.async-producer kernel and the TMA-producer kernel.
struct TcCtx {
    uint8_t* sW;
    uint8_t* sA;
    float* sEpi;
    ChunkInfo* sChunk;
    uint32_t bar0;       // full[NSTAGE], empty[NSTAGE]
    int nkb, stage_bytes, w_half;
    __device__ __forceinline__ uint32_t full_bar(int s) const { return bar0 + 8u * s; }
    __device__ __forceinline__ uint32_t empty_bar(int s) const { return bar0 + 8u * (NSTAGE + s); }
};

// =============================== consumers (2 warpgroups: wgmma + epilogue) ===============================
// cw: consumer warp 0..7; warpgroup cw / 4 owns rows [64 (cw / 4), 64 (cw / 4) + 64) of each tile, warp cw % 4 of it
// holds the accumulator rows [16 (cw % 4), 16 (cw % 4) + 16) of that half.

struct NoExtraMma {
    __device__ __forceinline__ void operator()(int, int, uint64_t, uint64_t) const {}
};

// Main loop fed by the ring: acc = A (p.K columns, canonical ring stages) @ W (resident at c.sW).  Each ring slot is
// released once the wgmma group that read it has retired; stage / phase carry the ring position across tiles.
// extra(kb, ks, da_hi, da_lo) is called after the products of each k16 step, inside the same wgmma group: it may issue
// further wgmmas that read the same A stage into another accumulator.
template <bool SPLIT, int NCH, typename Extra = NoExtraMma>
__device__ __forceinline__ void tc_mma_ring(float (&acc)[16 * NCH], const TcParams& p, const TcCtx& c, int wg, int lane, int& stage,
                                            uint32_t& phase, const Extra& extra = Extra{}) {
    const int nkb = c.nkb, stage_bytes = c.stage_bytes, w_half = c.w_half;
    const uint32_t sW_u = smem_u32(c.sW);
    const uint32_t w_sbo = (uint32_t)(p.K / 8) * 128;  // bytes between 8-column (n) groups of W
    constexpr uint32_t A_SBO = (KC / 8) * 128;         // bytes between 8-row groups of a stage
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(c.full_bar(stage), phase);
        wgmma_fence();
        const uint32_t a_hi = smem_u32(c.sA + stage * stage_bytes) + (uint32_t)wg * 8 * A_SBO;
        const int ksteps = min(2, (p.K - kb * KC) / 16);
        for (int ks = 0; ks < ((p.debug & 4) ? 0 : ksteps); ++ks) {
            const uint64_t da_hi = make_desc(a_hi + ks * 256, 128, A_SBO);
            const uint32_t wk = sW_u + (uint32_t)(kb * (KC / 8) + ks * 2) * 128;
            const uint64_t db_hi = make_desc(wk, 128, w_sbo);
            wgmma_bf16<NCH>(acc, da_hi, db_hi, (kb | ks) ? 1u : 0u);
            const uint64_t da_lo = make_desc(a_hi + STAGE_HALF + ks * 256, 128, A_SBO);
            if constexpr (SPLIT) {
                const uint64_t db_lo = make_desc(wk + w_half, 128, w_sbo);
                wgmma_bf16<NCH>(acc, da_lo, db_hi, 1u);
                wgmma_bf16<NCH>(acc, da_hi, db_lo, 1u);
            }
            extra(kb, ks, da_hi, da_lo);
        }
        wgmma_commit();
        // the group of the previous k block has retired: its ring slot is free (this one stays in flight)
        if (prev >= 0) {
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(c.empty_bar(prev));
        }
        prev = stage;
        if (++stage == p.nstage) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (lane == 0 && prev >= 0) mbar_arrive(c.empty_bar(prev));
    if (p.debug & 4) {
#pragma unroll
        for (int j = 0; j < 16 * NCH; ++j) acc[j] = 0.f;
    }
}

// Main loop from a resident operand: acc = A (this warpgroup's 64 x K tile at a_u, bf16 hi image, lo image a_half bytes
// further) @ W (K x 32 NCH image at w_u, lo image w_half bytes further), both canonical K-major.  The k16 steps and the
// three split-bf16 products run in the same order as in tc_mma_ring, so the result is bitwise that of the ring-fed loop.
// accumulate: continue the k sum already in acc (the k steps of a longer ring-fed loop that follow those in acc).
template <int NCH>
__device__ __forceinline__ void tc_mma_resident(float (&acc)[16 * NCH], uint32_t a_u, uint32_t a_half, int K, uint32_t w_u, uint32_t w_half,
                                                bool accumulate = false) {
    const uint32_t sbo = (uint32_t)(K / 8) * 128;  // A rows and W columns: 8-groups K / 8 core matrices apart
    wgmma_fence();
    for (int ks = 0; ks < K / 16; ++ks) {
        const uint64_t da_hi = make_desc(a_u + ks * 256, 128, sbo), da_lo = make_desc(a_u + a_half + ks * 256, 128, sbo);
        const uint64_t db_hi = make_desc(w_u + ks * 256, 128, sbo), db_lo = make_desc(w_u + w_half + ks * 256, 128, sbo);
        wgmma_bf16<NCH>(acc, da_hi, db_hi, (ks || accumulate) ? 1u : 0u);
        wgmma_bf16<NCH>(acc, da_lo, db_hi, 1u);
        wgmma_bf16<NCH>(acc, da_hi, db_lo, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
}

// Epilogue of one 64-row half tile from the accumulator registers: this warp's 16 rows, one 32-column chunk at a time,
// into the output segments of p (chunk table `chunks`, one entry per 32 columns of p).  DSILU = false compiles out the
// phi' epilogue (p.epi must then be AB2_EPI_NONE).  GENERIC = false compiles out the per-element path: every chunk must
// then be on the coalesced path (ChunkInfo::ok, checked by the caller's host code).  NL: the nonlinearity phi (AB2_NL_*).
template <typename TSrc, int NCH, bool DSILU = true, bool GENERIC = true, int NL = AB2_NL_SILU>
__device__ __forceinline__ void tc_epilogue(const TcParams& p, const ChunkInfo* chunks, float* stg, const float (&acc)[16 * NCH], int64_t tile,
                                            int wg, int w4, int lane) {
    {
        const int64_t m_base = tile * BM + wg * 64 + w4 * 16;
        const int64_t left64 = p.M - m_base;  // <= 0: this warp's rows lie beyond M
        const int rows_left = left64 >= 16 ? 16 : (left64 > 0 ? (int)left64 : 0);
        const int rsub = lane >> 3, c4 = lane & 7;
        // row handled in slot itr: itr*4 + rsub; loads of a partial tile read a clamped (valid) row
        auto row_of = [&](int itr) { const int r = itr * 4 + rsub; return r < rows_left ? r : rows_left - 1; };
        // generic path: 16 consecutive columns [c0, c0 + 16) of row m
        auto process = [&](int64_t m, int c0, const float (&vin)[16]) {
            float v[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = vin[j];
            if (DSILU && p.epi == AB2_EPI_MUL_DSILU) {
                const TSrc* ax = (const TSrc*)p.aux + m * p.aux_ld + c0;
                if (sizeof(TSrc) == 4 && c0 + 16 <= p.N && ((reinterpret_cast<uintptr_t>(ax) & 15) == 0)) {
                    const float4* a4 = reinterpret_cast<const float4*>(ax);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float4 x = __ldg(a4 + t);
                        v[4 * t] *= dact_f<NL>(x.x); v[4 * t + 1] *= dact_f<NL>(x.y); v[4 * t + 2] *= dact_f<NL>(x.z); v[4 * t + 3] *= dact_f<NL>(x.w);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (c0 + j < p.N) v[j] *= dact_f<NL>(to_acc<float>(ax[j]));
                }
            }
            // scatter the 16 columns into the output segments
            int seg_lo = 0;
#pragma unroll
            for (int s = 0; s < AB2_MAX_SEG; ++s) {
                if (s < p.n_o) {
                    const int seg_hi = seg_lo + p.o[s].width;
                    const int lo = max(seg_lo, c0), hi = min(seg_hi, min(c0 + 16, p.N));
                    if (lo < hi) {
                        TSrc* dst = (TSrc*)p.o[s].ptr + m * p.o[s].ld + (lo - seg_lo);
                        const bool vec = (sizeof(TSrc) == 4) && (hi - lo == 16) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
                        if (vec) {
                            float4* d4 = reinterpret_cast<float4*>(dst);
#pragma unroll
                            for (int t = 0; t < 4; ++t) {
                                float4 o4 = make_float4(v[4 * t], v[4 * t + 1], v[4 * t + 2], v[4 * t + 3]);
                                if (p.o[s].accum) {
                                    const float4 old = d4[t];
                                    o4.x += old.x; o4.y += old.y; o4.z += old.z; o4.w += old.w;
                                }
                                d4[t] = o4;
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < 16; ++j) {
                                const int n = c0 + j;
                                if (n >= lo && n < hi) {
                                    float x = v[j];
                                    if (p.o[s].accum) x += to_acc<float>(dst[n - lo]);
                                    dst[n - lo] = from_acc<TSrc>(x);
                                }
                            }
                        }
                    }
                    seg_lo = seg_hi;
                }
            }
        };
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
            const int c0 = ch * 32;
            // accumulator fragment -> staging rows (row = lane / 4 and lane / 4 + 8)
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int col = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(stg + (lane >> 2) * EPI_LD + col) = make_float2(acc[16 * ch + 4 * j], acc[16 * ch + 4 * j + 1]);
                *reinterpret_cast<float2*>(stg + ((lane >> 2) + 8) * EPI_LD + col) = make_float2(acc[16 * ch + 4 * j + 2], acc[16 * ch + 4 * j + 3]);
            }
            __syncwarp();
            const ChunkInfo ci = chunks[ch];
            if ((p.debug & 1) || rows_left == 0) {
            } else if (ci.ok) {
                // coalesced path: every global access covers 4 rows x 128 B.
                // 1) shared-memory reads, 2) (uniform) epilogue variants with all global loads issued before use,
                // 3) stores: tile base pointer + 32-bit row offsets.
                float4 x[4];
#pragma unroll
                for (int itr = 0; itr < 4; ++itr) x[itr] = *reinterpret_cast<const float4*>(stg + (itr * 4 + rsub) * EPI_LD + c4 * 4);
                float* tb = ci.optr + m_base * ci.ld + c4 * 4;
                const uint32_t ol = (uint32_t)ci.ld;
                uint32_t off[4];
#pragma unroll
                for (int itr = 0; itr < 4; ++itr) off[itr] = (uint32_t)row_of(itr) * ol;
                if (DSILU && p.epi == AB2_EPI_MUL_DSILU) {
                    float4 ax[4];
                    const float* ab = ci.aptr + m_base * p.aux_ld + c4 * 4;
                    const uint32_t al = (uint32_t)p.aux_ld;
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) ax[itr] = ldg128_nc(ab + (uint32_t)row_of(itr) * al);
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) {
                        x[itr].x *= dact_fast<NL>(ax[itr].x); x[itr].y *= dact_fast<NL>(ax[itr].y);
                        x[itr].z *= dact_fast<NL>(ax[itr].z); x[itr].w *= dact_fast<NL>(ax[itr].w);
                    }
                }
                if (ci.accum) {
                    float4 old[4];
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) old[itr] = ldg128(tb + off[itr]);
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) {
                        x[itr].x += old[itr].x; x[itr].y += old[itr].y; x[itr].z += old[itr].z; x[itr].w += old[itr].w;
                    }
                }
#pragma unroll
                for (int itr = 0; itr < 4; ++itr)
                    if (itr * 4 + rsub < rows_left) stg128(tb + off[itr], x[itr]);
            } else if constexpr (GENERIC) {
                // generic path: lane -> (row lane % 16, columns c0 + 16 (lane / 16) .. + 16)
                const int r = lane & 15, h = lane >> 4;
                if (r < rows_left && c0 + 16 * h < p.N) {
                    float v[16];
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float4 q = *reinterpret_cast<const float4*>(stg + r * EPI_LD + 16 * h + 4 * t);
                        v[4 * t] = q.x; v[4 * t + 1] = q.y; v[4 * t + 2] = q.z; v[4 * t + 3] = q.w;
                    }
                    process(m_base + r, c0 + 16 * h, v);
                }
            }
            __syncwarp();  // staging buffer is rewritten by the next chunk
        }
    }
}

template <typename TSrc, bool SPLIT, int NCH, int NL>
__device__ __forceinline__ void tc_consumer_role(const TcParams& p, const TcCtx& c, int cw, int lane) {
    const int wg = cw >> 2, w4 = cw & 3;
    float* stg = c.sEpi + cw * 16 * EPI_LD;
    int stage = 0;
    uint32_t phase = 0;
    float acc[16 * NCH];
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        tc_mma_ring<SPLIT, NCH>(acc, p, c, wg, lane, stage, phase);
        tc_epilogue<TSrc, NCH, true, true, NL>(p, c.sChunk, stg, acc, tile, wg, w4, lane);
    }
}

template <typename TSrc, bool SPLIT, int NCH, int NL>
__global__ void __launch_bounds__(NTHREADS, 1) linear_tc_kernel(const TcParams p) {
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // warp-uniform role index
    const int w_half = p.Npad * p.K * 2;                     // bytes of one W image
    const int w_bytes = SPLIT ? 2 * w_half : w_half;
    uint8_t* sW = smem;
    uint8_t* sA = smem + ((w_bytes + 127) & ~127);
    const int stage_bytes = SPLIT ? 2 * STAGE_HALF : STAGE_HALF;
    uint8_t* sRaw = sA + p.nstage * stage_bytes;
    const int raw_stage = RAW_STAGE * (p.has_aux ? 2 : 1);
    float* sEpi = reinterpret_cast<float*>(sRaw + p.raw_depth * raw_stage);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sEpi) + EPI_BYTES);  // full[NSTAGE], empty[NSTAGE]
    ChunkInfo* sChunk = reinterpret_cast<ChunkInfo*>(reinterpret_cast<uint8_t*>(bars) + TAIL_BARS);
    KEnt* sKmap = reinterpret_cast<KEnt*>(reinterpret_cast<uint8_t*>(sChunk) + TAIL_CHUNK);
    KEnt* sKaux = sKmap + MAX_K / 8;
    const uint32_t bar0 = smem_u32(bars);
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (NSTAGE + s); };

    // ---- one-time setup ----
    if (threadIdx.x == 0) {
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(full_bar(s), NPROD * 32);
            mbar_init(empty_bar(s), NCONS);  // one arrive per consumer warp once its wgmma reads of the slot retired
        }
        fence_barrier_init();
    }
    if (threadIdx.x < MAX_K / 8) {
        // k-chunk tables: which A segment (and aux segment) holds concat columns [8e, 8e+8)
        const int e = threadIdx.x;
        KEnt ent{nullptr, 0}, aent{nullptr, 0};
        int kk = e * 8;
        bool found = kk >= p.K;
#pragma unroll
        for (int sgi = 0; sgi < AB2_MAX_SEG; ++sgi) {
            if (sgi < p.n_a && !found) {
                if (kk < p.a[sgi].width) {
                    ent.ptr = (const TSrc*)p.a[sgi].ptr + kk;
                    ent.ld = p.a[sgi].ld;
                    if (p.a[sgi].aux) {
                        aent.ptr = (const TSrc*)p.a[sgi].aux + kk;
                        aent.ld = p.a[sgi].aux_ld;
                    }
                    found = true;
                }
                kk -= p.a[sgi].width;
            }
        }
        sKmap[e] = ent;
        sKaux[e] = aent;
    } else if (threadIdx.x < MAX_K / 8 + MAX_CHUNK) {
        sChunk[threadIdx.x - MAX_K / 8] = tc_chunk_info<TSrc>(p, (threadIdx.x - MAX_K / 8) * 32);
    }
    // stage W (pre-packed canonical images of this column slice) with plain 16-byte copies
    {
        const uint4* src = reinterpret_cast<const uint4*>(p.Wpacked);
        uint4* dst = reinterpret_cast<uint4*>(sW);
        for (int e = threadIdx.x; e < w_half / 16; e += NTHREADS) dst[e] = __ldg(src + e);
        if constexpr (SPLIT) {
            const uint4* srcl = reinterpret_cast<const uint4*>(p.Wlo);
            uint4* dstl = reinterpret_cast<uint4*>(sW + w_half);
            for (int e = threadIdx.x; e < w_half / 16; e += NTHREADS) dstl[e] = __ldg(srcl + e);
        }
    }
    fence_proxy_async();  // W was written through the generic proxy, wgmma reads via the async proxy
    __syncthreads();

    const int nkb = (p.K + KC - 1) / KC;
    TcCtx ctx;
    ctx.sW = sW; ctx.sA = sA; ctx.sEpi = sEpi; ctx.sChunk = sChunk; ctx.bar0 = bar0;
    ctx.nkb = nkb; ctx.stage_bytes = stage_bytes; ctx.w_half = w_half;

    if (warp < NPROD) {
        // =============================== producers ===============================
        // 16 row-groups of 8 rows per stage, 2 per warp; lane -> (row in group, 8-wide k chunk).
        // Register double buffering: the loads of work item s+1 are in flight while item s is
        // converted and stored, and while this warp waits for its ring slot.
        constexpr int GPW = 16 / NPROD;  // row groups per warp per stage
        const int r8 = lane & 7, kc = lane >> 3;
        const int64_t my_tiles = (p.num_tiles > blockIdx.x) ? (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        const int64_t total = my_tiles * nkb;
        int stage = 0;
        uint32_t phase = 0;
        constexpr int CH = (sizeof(TSrc) == 4) ? 2 : 1;  // 16-byte chunks per 8 elements
        const uint32_t raw_u = smem_u32(sRaw);
        // Cursors of the next work item to issue / to fetch (tile, k block, raw slot): plain counters,
        // no 64-bit div/mod per item.
        int64_t i_tile = blockIdx.x, i_seq = 0;
        int i_kb = 0, i_slot = 0, f_kb = 0, f_slot = 0;
        // issue the asynchronous copies of the next work item into this thread's private raw slot
        auto issue = [&]() {
            if (i_seq < total) {
                const int64_t row0 = i_tile * BM;
                const int64_t left = p.M - row0;
                const int rows_left = left < BM ? (int)left : BM;
                const KEnt e = sKmap[i_kb * (KC / 8) + kc];
                const bool kok = e.ptr != nullptr && !(p.debug & 2);
                const uint8_t* tb = reinterpret_cast<const uint8_t*>(e.ptr) + row0 * e.ld * (int64_t)sizeof(TSrc);
                const uint32_t pitch = (uint32_t)e.ld * (uint32_t)sizeof(TSrc);
                KEnt ea{nullptr, 0};
                if (p.has_aux) ea = sKaux[i_kb * (KC / 8) + kc];
                const uint8_t* tba = reinterpret_cast<const uint8_t*>(ea.ptr) + row0 * ea.ld * (int64_t)sizeof(TSrc);
                const uint32_t pitch_a = (uint32_t)ea.ld * (uint32_t)sizeof(TSrc);
#pragma unroll
                for (int i = 0; i < GPW; ++i) {
                    const int row = (warp * GPW + i) * 8 + r8;
                    const bool inb = kok && row < rows_left;
                    const uint8_t* src = tb + (uint32_t)row * pitch;
#pragma unroll
                    for (int h = 0; h < CH; ++h) {
                        const uint32_t dst = raw_u + (uint32_t)(i_slot * raw_stage + ((i * CH + h) * 256 + threadIdx.x) * 16);
                        cp_async16(dst, inb ? (const void*)(src + 16 * h) : p.Wpacked, inb ? 16u : 0u);  // src-size 0 -> zero fill
                    }
                    if (p.has_aux) {
                        const bool ain = inb && ea.ptr != nullptr;
                        const uint8_t* ax = tba + (uint32_t)row * pitch_a;
#pragma unroll
                        for (int h = 0; h < CH; ++h) {
                            const uint32_t dst = raw_u + (uint32_t)(i_slot * raw_stage + ((4 + i * CH + h) * 256 + threadIdx.x) * 16);
                            cp_async16(dst, ain ? (const void*)(ax + 16 * h) : p.Wpacked, ain ? 16u : 0u);
                        }
                    }
                }
            }
            cp_async_commit();  // always commit so that group counting stays uniform
            ++i_seq;
            if (++i_slot == p.raw_depth) i_slot = 0;
            if (++i_kb == nkb) { i_kb = 0; i_tile += gridDim.x; }
        };
        auto fetch = [&](float (&v)[GPW][8]) {
            const uint8_t* base = sRaw + f_slot * raw_stage;
            auto rd8 = [&](int chunk0, float (&o)[8]) {
                if constexpr (sizeof(TSrc) == 4) {
                    const float4 x = *reinterpret_cast<const float4*>(base + ((chunk0 + 0) * 256 + threadIdx.x) * 16);
                    const float4 y = *reinterpret_cast<const float4*>(base + ((chunk0 + 1) * 256 + threadIdx.x) * 16);
                    o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w; o[4] = y.x; o[5] = y.y; o[6] = y.z; o[7] = y.w;
                } else {
                    const uint4 x = *reinterpret_cast<const uint4*>(base + (chunk0 * 256 + threadIdx.x) * 16);
                    const __nv_bfloat162* hh = reinterpret_cast<const __nv_bfloat162*>(&x);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float2 f = __bfloat1622float2(hh[t]);
                        o[2 * t] = f.x; o[2 * t + 1] = f.y;
                    }
                }
            };
            // segments without an aux matrix have zero-filled aux chunks; they must not scale A
            const bool has = p.has_aux && sKaux[f_kb * (KC / 8) + kc].ptr != nullptr;
#pragma unroll
            for (int i = 0; i < GPW; ++i) {
                rd8(i * CH, v[i]);
                if (p.has_aux) {
                    float w[8];
                    rd8(4 + i * CH, w);
                    if (has) {
#pragma unroll
                        for (int t = 0; t < 8; ++t) v[i][t] *= dact_fast<NL>(w[t]);
                    }
                }
            }
            if (++f_slot == p.raw_depth) f_slot = 0;
            if (++f_kb == nkb) f_kb = 0;
        };
        auto emit = [&](float (&v)[GPW][8]) {
            mbar_wait(empty_bar(stage), phase ^ 1);
            uint8_t* st_hi = sA + stage * stage_bytes;
#pragma unroll
            for (int i = 0; i < GPW; ++i) {
                if (p.act == AB2_ACT_SILU) {
#pragma unroll
                    for (int t = 0; t < 8; ++t) v[i][t] = act_fast<NL>(v[i][t]);
                }
                const int g = warp * GPW + i;
                const uint32_t off = g * (KC / 8) * 128 + kc * 128 + r8 * 16;
                uint32_t hi[4];
                float lo[8];
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const __nv_bfloat16 h0 = __float2bfloat16_rn(v[i][2 * t]), h1 = __float2bfloat16_rn(v[i][2 * t + 1]);
                    lo[2 * t] = v[i][2 * t] - __bfloat162float(h0);
                    lo[2 * t + 1] = v[i][2 * t + 1] - __bfloat162float(h1);
                    __nv_bfloat162 hh;
                    hh.x = h0; hh.y = h1;
                    hi[t] = *reinterpret_cast<uint32_t*>(&hh);
                }
                *reinterpret_cast<uint4*>(st_hi + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                if constexpr (SPLIT) {
                    *reinterpret_cast<uint4*>(st_hi + STAGE_HALF + off) =
                        make_uint4(pack_bf16x2(lo[0], lo[1]), pack_bf16x2(lo[2], lo[3]), pack_bf16x2(lo[4], lo[5]), pack_bf16x2(lo[6], lo[7]));
                }
            }
            fence_proxy_async();
            mbar_arrive(full_bar(stage));
            if (++stage == p.nstage) { stage = 0; phase ^= 1; }
        };
        static_assert(GPW == 2, "raw slot layout assumes 2 row groups per producer warp");
        for (int d = 0; d < p.raw_depth; ++d) issue();
        for (int64_t seq = 0; seq < total; ++seq) {
            if (p.raw_depth == 4) cp_async_wait<3>();  // the oldest group (= item seq) has landed
            else cp_async_wait<1>();
            float v[GPW][8];
            fetch(v);
            issue();          // item seq + raw_depth refills the slot just drained
            emit(v);
        }
        cp_async_wait<0>();
    } else {
        tc_consumer_role<TSrc, SPLIT, NCH, NL>(p, ctx, warp - NPROD, lane);
    }
}

// =========================================================================================
// TMA-producer variant (fp32 storage, every A segment a multiple of 32 columns wide).
//
//   warps 0-7    : four converter GROUPS of two warps.  Group g owns the stages q = g (mod 4) and the raw slots that feed
//                  them.  One elected lane of the group issues cp.async.bulk.tensor.2d loads (SASS UTMALDG) of 128-row x
//                  32-column fp32 boxes (16 KB, SWIZZLE_128B) into its raw slots, one box per k-chunk (+ one for the
//                  silu' multiplier of that chunk), completing on an mbarrier; rows beyond M are zero-filled by the TMA
//                  unit.  The group waits for the raw slot, reads it conflict-free (the 128-byte swizzle puts the 8 rows
//                  of a core matrix in 8 different bank groups), refills it NR sequence numbers ahead once all its warps
//                  have drained it, applies SiLU / silu'(aux), splits into bf16 hi + lo and writes the canonical
//                  K-major stage.  Four stages are in conversion at once, so the fixed latency of one stage (mbarrier
//                  wait, LDS, convert, STS, fence.proxy.async, arrive) does not bound the load rate.  No separate TMA
//                  warp: a 17th warp would cost the consumers their 128-register budget.
//   warps 8-15   : consumers, unchanged (tc_consumer_role).
// =========================================================================================
constexpr int TMA_BOX_BYTES = BM * KC * 4;  // 16 KB

struct alignas(64) TmaMaps {
    CUtensorMap a[AB2_MAX_SEG];
    CUtensorMap x[AB2_MAX_SEG];
};

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
                 "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(x), "r"(y)
                 : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}

// bf16 hi + lo split of two fp32 values (hi = rn(x), lo = rn(x - hi)), packed as bf16x2 pairs
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    const __nv_bfloat16 h0 = __float2bfloat16_rn(a), h1 = __float2bfloat16_rn(b);
    __nv_bfloat162 hh;
    hh.x = h0; hh.y = h1;
    hi = *reinterpret_cast<uint32_t*>(&hh);
    lo = pack_bf16x2(a - __bfloat162float(h0), b - __bfloat162float(h1));
}

// barriers of the TMA-fed ring: canonical full / empty [NSTAGE] at bar0, raw-slot full [8] at rbar0
__device__ __forceinline__ void tma_init_bars(uint32_t bar0, uint32_t rbar0, int wpg) {
    for (int s = 0; s < NSTAGE; ++s) {
        mbar_init(bar0 + 8u * s, wpg * 32);          // canonical stage full: the warps of one converter group
        mbar_init(bar0 + 8u * (NSTAGE + s), NCONS);  // empty: one arrive per consumer warp
    }
    for (int s = 0; s < 8; ++s) mbar_init(rbar0 + 8u * s, 1);  // expect_tx arrive of the issuing lane
    fence_barrier_init();
}

// k-chunk table entry i (concat columns [32 i, 32 i + 32)): segment index, column offset inside the segment, has-aux flag
__device__ __forceinline__ int4 tma_kseg_entry(const TcParams& p, int i) {
    int kk = i * KC;
    int4 ent = make_int4(-1, 0, 0, 0);
#pragma unroll
    for (int sgi = 0; sgi < AB2_MAX_SEG; ++sgi) {
        if (sgi < p.n_a && ent.x < 0 && kk < p.K) {
            if (kk < p.a[sgi].width) ent = make_int4(sgi, kk, p.a[sgi].aux ? 1 : 0, 0);
            kk -= p.a[sgi].width;
        }
    }
    return ent;
}

// copy the hi and lo images (w_half bytes each) of a packed W into shared memory, all threads of the CTA
__device__ __forceinline__ void stage_w(uint8_t* dst, const void* hi, const void* lo, int w_half) {
    const uint4* src = reinterpret_cast<const uint4*>(hi);
    uint4* d = reinterpret_cast<uint4*>(dst);
    for (int e = threadIdx.x; e < w_half / 16; e += NTHREADS) d[e] = __ldg(src + e);
    const uint4* srcl = reinterpret_cast<const uint4*>(lo);
    uint4* dl = reinterpret_cast<uint4*>(dst + w_half);
    for (int e = threadIdx.x; e < w_half / 16; e += NTHREADS) dl[e] = __ldg(srcl + e);
}

// Converter warps 0-7 (G groups) of the TMA-fed ring: total = work items (tile, k block) of this CTA, sKseg the k-chunk
// table, rbar0 the raw-slot barriers.
// G converter groups of 8/G warps.  A raw slot and a canonical stage must always be consumed / produced by the SAME group
// (NR % G == 0 and nstage % G == 0, checked on the host): a group then never waits more than one mbarrier phase ahead
// of its own slot.  (With slots shared between groups a group's first wait can be for the SECOND fill of a slot whose
// first fill has not completed yet -- the parity wait returns immediately and the pipeline falls apart.)
template <int G, int NL>
__device__ __forceinline__ void tma_converter_role(const TcParams& p, const TmaMaps& maps, int NR, const TcCtx& ctx, uint8_t* sRaw,
                                                   const int4* sKseg, uint32_t rbar0, int64_t total, int warp, int lane) {
    constexpr int WPG = NPROD / G;      // warps per converter group
    constexpr int RGW = 16 / WPG;       // 8-row groups of a stage handled by one warp
    const int nkb = ctx.nkb;
    const int raw_slot = TMA_BOX_BYTES * (p.has_aux ? 2 : 1);
    uint8_t* sA = ctx.sA;
    const int stage_bytes = ctx.stage_bytes;
    auto rfull_bar = [&](int s) { return rbar0 + 8u * s; };

    // loads of sequence number qs (k block qs % nkb of this CTA's tile qs / nkb) into raw slot rs
    auto tma_issue = [&](int64_t qs, int rs) {
        const int64_t tile = blockIdx.x + (qs / nkb) * gridDim.x;
        const int4 ent = sKseg[(int)(qs % nkb)];
        const uint32_t dst = smem_u32(sRaw + (size_t)rs * raw_slot);
        const bool ax = p.has_aux && ent.z;
        mbar_expect_tx(rfull_bar(rs), TMA_BOX_BYTES * (ax ? 2u : 1u));
        if (!(p.debug & 2)) {
            tma_load_2d(dst, &maps.a[ent.x], ent.y, (int)(tile * BM), rfull_bar(rs));
            if (ax) tma_load_2d(dst + TMA_BOX_BYTES, &maps.x[ent.x], ent.y, (int)(tile * BM), rfull_bar(rs));
        } else {
            asm volatile("mbarrier.complete_tx.shared::cta.b64 [%0], %1;" ::"r"(rfull_bar(rs)), "r"(TMA_BOX_BYTES * (ax ? 2u : 1u)) : "memory");
        }
    };

    {
        // =============================== converters ===============================
        const int grp = warp / WPG, sub = warp % WPG;
        const int r8 = lane & 7, kc = lane >> 3;
        // raw slot / canonical stage of sequence number qs: plain counters (advance by G per iteration)
        int rs = grp % NR, cs = grp % p.nstage, kb = grp % nkb;
        uint32_t rph = (uint32_t)((grp / NR) & 1), cph = (uint32_t)((grp / p.nstage) & 1);
        const bool leader = sub == 0 && lane == 0;
        if (leader) {
            for (int sgi = 0; sgi < p.n_a; ++sgi) {
                asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.a[sgi])) : "memory");
                if (p.a[sgi].aux) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.x[sgi])) : "memory");
            }
            for (int q = grp; q < NR && q < total; q += G) tma_issue(q, q);  // first fill of this group's raw slots
        }
        for (int64_t qs = grp; qs < total; qs += G) {
            mbar_wait(rfull_bar(rs), rph);
            const uint8_t* raw = sRaw + (size_t)rs * raw_slot;
            const bool ax = p.has_aux && sKseg[kb].z;
            float v[RGW][8];
#pragma unroll
            for (int i = 0; i < RGW; ++i) {
                const int row = (sub * RGW + i) * 8 + r8;
                const uint8_t* rp = raw + row * 128;
                const float4 x = *reinterpret_cast<const float4*>(rp + (((2 * kc) ^ r8) << 4));
                const float4 y = *reinterpret_cast<const float4*>(rp + (((2 * kc + 1) ^ r8) << 4));
                v[i][0] = x.x; v[i][1] = x.y; v[i][2] = x.z; v[i][3] = x.w; v[i][4] = y.x; v[i][5] = y.y; v[i][6] = y.z; v[i][7] = y.w;
            }
            if (ax) {
#pragma unroll
                for (int i = 0; i < RGW; ++i) {
                    const int row = (sub * RGW + i) * 8 + r8;
                    const uint8_t* rp = raw + TMA_BOX_BYTES + row * 128;
                    const float4 x = *reinterpret_cast<const float4*>(rp + (((2 * kc) ^ r8) << 4));
                    const float4 y = *reinterpret_cast<const float4*>(rp + (((2 * kc + 1) ^ r8) << 4));
                    v[i][0] *= dact_fast<NL>(x.x); v[i][1] *= dact_fast<NL>(x.y); v[i][2] *= dact_fast<NL>(x.z); v[i][3] *= dact_fast<NL>(x.w);
                    v[i][4] *= dact_fast<NL>(y.x); v[i][5] *= dact_fast<NL>(y.y); v[i][6] *= dact_fast<NL>(y.z); v[i][7] *= dact_fast<NL>(y.w);
                }
            }
            // raw slot drained by every warp of the group (values are in registers): refill it
            asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(WPG * 32) : "memory");
            if (leader && qs + NR < total) tma_issue(qs + NR, rs);
            mbar_wait(ctx.empty_bar(cs), cph ^ 1);
            uint8_t* st_hi = sA + cs * stage_bytes;
#pragma unroll
            for (int i = 0; i < RGW; ++i) {
                if (p.act == AB2_ACT_SILU) {
#pragma unroll
                    for (int t = 0; t < 8; ++t) v[i][t] = act_fast<NL>(v[i][t]);
                }
                const int g = sub * RGW + i;
                const uint32_t off = g * (KC / 8) * 128 + kc * 128 + r8 * 16;
                uint32_t hi[4];
                float lo[8];
#pragma unroll
                for (int t = 0; t < 4; ++t) {
                    const __nv_bfloat16 h0 = __float2bfloat16_rn(v[i][2 * t]), h1 = __float2bfloat16_rn(v[i][2 * t + 1]);
                    lo[2 * t] = v[i][2 * t] - __bfloat162float(h0);
                    lo[2 * t + 1] = v[i][2 * t + 1] - __bfloat162float(h1);
                    __nv_bfloat162 hh;
                    hh.x = h0; hh.y = h1;
                    hi[t] = *reinterpret_cast<uint32_t*>(&hh);
                }
                *reinterpret_cast<uint4*>(st_hi + off) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4*>(st_hi + STAGE_HALF + off) =
                    make_uint4(pack_bf16x2(lo[0], lo[1]), pack_bf16x2(lo[2], lo[3]), pack_bf16x2(lo[4], lo[5]), pack_bf16x2(lo[6], lo[7]));
            }
            fence_proxy_async();
            mbar_arrive(ctx.full_bar(cs));
            // advance the counters by G stages (NR and nstage are multiples of G: at most one wrap each)
            rs += G; if (rs >= NR) { rs -= NR; rph ^= 1; }
            cs += G; if (cs >= p.nstage) { cs -= p.nstage; cph ^= 1; }
            kb += G; while (kb >= nkb) kb -= nkb;
        }
    }
}

template <int G, int NCH, int NL>
__global__ void __launch_bounds__(NTHREADS, 1) linear_tma_kernel(const TcParams p, const __grid_constant__ TmaMaps maps, int NR) {
    constexpr int WPG = NPROD / G;      // warps per converter group
    using TSrc = float;
    constexpr bool SPLIT = true;
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // warp-uniform role index
    const int w_half = p.Npad * p.K * 2;
    const int w_bytes = 2 * w_half;
    const int stage_bytes = 2 * STAGE_HALF;
    const int raw_slot = TMA_BOX_BYTES * (p.has_aux ? 2 : 1);
    // plan: raw ring (1024-byte aligned, swizzle atom) | W | canonical ring | epilogue staging | prefetch | tail
    uint8_t* sRaw = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);
    uint8_t* sW = sRaw + (size_t)NR * raw_slot;
    uint8_t* sA = sW + ((w_bytes + 127) & ~127);
    float* sEpi = reinterpret_cast<float*>(sA + p.nstage * stage_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sEpi) + EPI_BYTES);
    ChunkInfo* sChunk = reinterpret_cast<ChunkInfo*>(reinterpret_cast<uint8_t*>(bars) + TAIL_BARS);
    // k-chunk table (one entry per 32 columns): segment index, column offset inside the segment, has-aux flag
    int4* sKseg = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(sChunk) + TAIL_CHUNK);
    uint64_t* rbars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sKseg) + (MAX_K / 32) * 16);  // raw_full[8]
    const uint32_t bar0 = smem_u32(bars), rbar0 = smem_u32(rbars);
    const int nkb = p.K / KC;

    // ---- one-time setup ----
    if (threadIdx.x == 0) tma_init_bars(bar0, rbar0, WPG);
    if (threadIdx.x < MAX_K / 32) {
        sKseg[threadIdx.x] = tma_kseg_entry(p, threadIdx.x);
    } else if (threadIdx.x >= 64 && threadIdx.x < 64 + MAX_CHUNK) {
        sChunk[threadIdx.x - 64] = tc_chunk_info<TSrc>(p, (threadIdx.x - 64) * 32);
    }
    stage_w(sW, p.Wpacked, p.Wlo, w_half);
    fence_proxy_async();
    __syncthreads();
    TcCtx ctx;
    ctx.sW = sW; ctx.sA = sA; ctx.sEpi = sEpi; ctx.sChunk = sChunk; ctx.bar0 = bar0;
    ctx.nkb = nkb; ctx.stage_bytes = stage_bytes; ctx.w_half = w_half;
    const int64_t my_tiles = (p.num_tiles > blockIdx.x) ? (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int64_t total = my_tiles * nkb;

    if (warp >= NPROD) {
        tc_consumer_role<TSrc, SPLIT, NCH, NL>(p, ctx, warp - NPROD, lane);
    } else {
        tma_converter_role<G, NL>(p, maps, NR, ctx, sRaw, sKseg, rbar0, total, warp, lane);
    }
}

// =========================================================================================
// Hidden-layer gradient GEMM of the scalar-embed MLP and the radial adjoint in one kernel (ab2_radial_pq_bwd_gemm).  With
// the radial embedding folded into that MLP's first layer (radial.cu, PQ form) its pre-activation is
// h[z][c] = sum_n B_n(x_z) PQ[pair_z][n][c], and its backward ends in
//   g_h = Gout @ W2^T                                                                     (ab2_linear, N = H)
//   gvec[z] += sum_c g_h[z][c] phi'(h[z][c]) sum_n dB_n(x_z) PQ[pair_z][n][c] * r_vec / (r_max |r|)   (radial_pq_bwd_kernel)
// Here the GEMM is that of linear_tma_kernel (converter warps, ring and main loop as they are) and the accumulator goes
// into the adjoint instead of to HBM.  Each consumer thread holds rows r8 and r8 + 8 of its warp's 16, 16 columns of each
// (fragment layout at wgmma_bf16), and per tile
//   - reads vec and the type pair of both rows (ctr / nbr one tile ahead, so the types gather does not wait on them);
//   - evaluates the radial basis, two of the eight functions per lane of the quad, shared by shuffles;
//   - recomputes its h columns with the fmaf chain of radial_pq_fwd_kernel (n order), so phi'(h) is that of the stored h;
//   - sums g_h phi'(h) sum_n dB_n PQ over its columns in the arithmetic of radial_pq_bwd_kernel, and the quad's four
//     partial sums with two xor shuffles;
//   - lane 0 of the quad, the only writer of the row, adds the row's gvec: no atomics, the result does not depend on
//     the launch.
// Neither g_h nor h reaches HBM.  PQ of every type pair (T^2 x 8 x H floats) is staged in the epilogue staging area,
// which this kernel does not otherwise use.
// =========================================================================================
constexpr int RADJ_NB = 8;  // Bessel functions of the PQ form

struct RadialAdjParams {
    const float* vec;         // [M][3]
    const int32_t* ctr;       // [M]
    const int32_t* nbr;       // [M]
    const int32_t* types;     // per atom
    const float* rmax_table;  // [T][T]
    const float* bw;          // [RADJ_NB] Bessel weights
    const float* PQ;          // [T * T][RADJ_NB][H]
    float* gvec;              // [M][3], accumulated into
    int num_types;
    float p;                  // polynomial cutoff order
};

template <int NCH, int NL>
__device__ __forceinline__ void radial_adjoint_consumer_role(const TcParams& p, const TcCtx& c, const RadialAdjParams& ra, const float* sPQ, int cw,
                                                             int lane) {
    constexpr int H = 32 * NCH;
    const int wg = cw >> 2, w4 = cw & 3;
    const int r8 = lane >> 2, cq = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    float acc[16 * NCH];
    // row i (0, 1) of this thread in a tile, clamped to the last edge: rows beyond M read valid data and write nothing
    auto row = [&](int64_t tile, int i) {
        const int64_t m = tile * BM + wg * 64 + w4 * 16 + r8 + 8 * i;
        return m < p.M ? m : p.M - 1;
    };
    int nc[2], nn[2];  // centre and neighbour of the rows of the next tile
    auto fetch_idx = [&](int64_t tile) {
        if (tile < p.num_tiles) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                nc[i] = __ldg(ra.ctr + row(tile, i));
                nn[i] = __ldg(ra.nbr + row(tile, i));
            }
        }
    };
    fetch_idx(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        int pair[2];
        float v[2][3];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            pair[i] = __ldg(ra.types + nc[i]) * ra.num_types + __ldg(ra.types + nn[i]);
            const float* vr = ra.vec + row(tile, i) * 3;
            v[i][0] = __ldg(vr); v[i][1] = __ldg(vr + 1); v[i][2] = __ldg(vr + 2);
        }
        fetch_idx(tile + gridDim.x);
        tc_mma_ring<true, NCH>(acc, p, c, wg, lane, stage, phase);  // acc = g_h of this thread's fragment
        float f[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const float r = sqrtf(v[i][0] * v[i][0] + v[i][1] * v[i][1] + v[i][2] * v[i][2]);
            const float rmax = __ldg(ra.rmax_table + pair[i]);
            float Bq[2], dBq[2];
            bessel_basis<float, true>(r / rmax, ra.p, 2, ra.bw + cq, Bq, dBq);  // functions cq, cq + 1
            float B[RADJ_NB], dB[RADJ_NB];
#pragma unroll
            for (int n = 0; n < RADJ_NB; ++n) {
                B[n] = __shfl_sync(0xffffffffu, Bq[n & 1], (lane & ~3) | (n >> 1));
                dB[n] = __shfl_sync(0xffffffffu, dBq[n & 1], (lane & ~3) | (n >> 1));
            }
            const float* m = sPQ + pair[i] * RADJ_NB * H + cq;
            float gx = 0.f;
#pragma unroll
            for (int j = 0; j < 4 * NCH; ++j) {  // columns 8 j + cq, 8 j + cq + 1
                float2 pq[RADJ_NB];
#pragma unroll
                for (int n = 0; n < RADJ_NB; ++n) pq[n] = *reinterpret_cast<const float2*>(m + n * H + 8 * j);
                float h0 = 0.f, h1 = 0.f, s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int n = 0; n < RADJ_NB; ++n) {
                    h0 = fmaf(B[n], pq[n].x, h0);
                    h1 = fmaf(B[n], pq[n].y, h1);
                    s0 = fmaf(dB[n], pq[n].x, s0);
                    s1 = fmaf(dB[n], pq[n].y, s1);
                }
                gx = fmaf(acc[4 * j + 2 * i] * dact_f<NL>(h0), s0, gx);
                gx = fmaf(acc[4 * j + 2 * i + 1] * dact_f<NL>(h1), s1, gx);
            }
            gx += __shfl_xor_sync(0xffffffffu, gx, 1);
            gx += __shfl_xor_sync(0xffffffffu, gx, 2);
            f[i] = gx / (rmax * r);  // dx/dr_vec = r_vec / (|r| r_max)
        }
        if ((lane & 3) == 0) {
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int64_t m = tile * BM + wg * 64 + w4 * 16 + r8 + 8 * i;
                if (m < p.M) {
                    float* g = ra.gvec + m * 3;
                    g[0] += f[i] * v[i][0];
                    g[1] += f[i] * v[i][1];
                    g[2] += f[i] * v[i][2];
                }
            }
        }
    }
}

template <int G, int NCH, int NL>
__global__ void __launch_bounds__(NTHREADS, 1) radial_adjoint_tma_kernel(const TcParams p, const __grid_constant__ TmaMaps maps, int NR,
                                                                         const RadialAdjParams ra) {
    constexpr int WPG = NPROD / G;  // warps per converter group
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // warp-uniform role index
    const int w_half = p.Npad * p.K * 2;
    const int w_bytes = 2 * w_half;
    const int stage_bytes = 2 * STAGE_HALF;
    // the plan of linear_tma_kernel without silu' multiplier (one box per raw slot); PQ in the epilogue staging area
    uint8_t* sRaw = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);
    uint8_t* sW = sRaw + (size_t)NR * TMA_BOX_BYTES;
    uint8_t* sA = sW + ((w_bytes + 127) & ~127);
    float* sPQ = reinterpret_cast<float*>(sA + p.nstage * stage_bytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sPQ) + EPI_BYTES);
    int4* sKseg = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(bars) + TAIL_BARS + TAIL_CHUNK);
    uint64_t* rbars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sKseg) + (MAX_K / 32) * 16);  // raw_full[8]
    const uint32_t bar0 = smem_u32(bars), rbar0 = smem_u32(rbars);
    const int nkb = p.K / KC;

    // ---- one-time setup ----
    if (threadIdx.x == 0) tma_init_bars(bar0, rbar0, WPG);
    if (threadIdx.x < MAX_K / 32) sKseg[threadIdx.x] = tma_kseg_entry(p, threadIdx.x);
    const int n_pq = ra.num_types * ra.num_types * RADJ_NB * 32 * NCH;
    for (int e = threadIdx.x; e < n_pq; e += NTHREADS) sPQ[e] = __ldg(ra.PQ + e);
    stage_w(sW, p.Wpacked, p.Wlo, w_half);
    fence_proxy_async();
    __syncthreads();
    TcCtx ctx;
    ctx.sW = sW; ctx.sA = sA; ctx.sEpi = sPQ; ctx.sChunk = nullptr; ctx.bar0 = bar0;
    ctx.nkb = nkb; ctx.stage_bytes = stage_bytes; ctx.w_half = w_half;
    const int64_t my_tiles = (p.num_tiles > blockIdx.x) ? (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    if (warp >= NPROD) {
        radial_adjoint_consumer_role<NCH, NL>(p, ctx, ra, sPQ, warp - NPROD, lane);
    } else {
        // the ring carries Gout as it is (p.act == AB2_ACT_NONE): the converters take no nonlinearity
        tma_converter_role<G, AB2_NL_SILU>(p, maps, NR, ctx, sRaw, sKseg, rbar0, my_tiles * nkb, warp, lane);
    }
}

// =========================================================================================
// Radial embedding and the scalar-embed MLP's folded last layer in one kernel (ab2_radial_embed_fwd): the forward of
//   h = radial_pq_fwd(vec)  [M][H]                                                         (radial_pq_fwd_kernel)
//   [w0 | x_0 | omega_0] = phi(h) @ W_fold   [M][N]                                         (ab2_linear, N / 128 slices)
// without h in memory, and with the whole output formed from one on-chip A tile instead of one pass over h per slice.
//   warps 0-7    : generators.  Thread t of the 256 owns row 16 (t / 32) + (t % 16) of each 128-row tile and half
//                  (t % 32) / 16 of its H / 8 core-matrix columns: it evaluates the row's basis (vec, ctr, nbr one tile
//                  ahead), forms h with the fmaf chain of radial_pq_fwd_kernel (n order from 0, so h is bitwise the
//                  stored one), applies phi as the converters do and writes the bf16 hi + lo split, one 16-byte store per
//                  image and core-matrix row, into a double-buffered canonical K-major [128][H] tile.  Each aligned
//                  group of 8 lanes writes one whole core matrix: conflict-free.
//   warps 8-15   : two consumer warpgroups.  Per tile and column chunk (the slicing of ab2_linear, so the same wgmma
//                  shapes) acc = phi(h) @ W_fold[:, chunk] from the resident tile in the k16 / split-product order of
//                  tc_mma_ring, then tc_epilogue into the chunk's output segments: bitwise the sliced launches' result.
//                  The A buffer is released once the last chunk's wgmma group has retired.
// W_fold (hi + lo) and PQ of every type pair stay resident.  PQ rows of consecutive pairs are 16 bytes further apart than
// 8 H floats, so that generator lanes of different pairs read different bank groups.
// =========================================================================================
constexpr int REMB_MAX_CHUNKS = 2;  // N <= 256 in column chunks of <= MAX_N

struct RadialEmbedParams {
    TcParams s[REMB_MAX_CHUNKS];  // per column chunk: M, N, Npad, output segments
    int n0[REMB_MAX_CHUNKS];      // first column of each chunk
    int n_chunks;
    int w_half;                   // bytes of the whole W_fold hi image (= lo image)
    const void* W;                // packed W_fold: hi image, then lo image
    const float* vec;             // [M][3]
    const int32_t* ctr;
    const int32_t* nbr;
    const int32_t* types;
    const float* rmax_table;      // [T][T]
    const float* bw;              // [RADJ_NB]
    const float* PQ;              // [T * T][RADJ_NB][H]
    int num_types;
    float p;                      // polynomial cutoff order
    int64_t M, num_tiles;
};

template <int NCH>
__device__ __forceinline__ void radial_embed_chunk(const TcParams& pc, const ChunkInfo* chunks, float* stg, uint32_t a_u, uint32_t a_half, int H,
                                                   uint32_t w_u, uint32_t w_half, bool release, uint32_t empty, int64_t tile, int wg, int w4,
                                                   int lane) {
    float acc[16 * NCH];
    tc_mma_resident<NCH>(acc, a_u, a_half, H, w_u, w_half);
    if (release && lane == 0) mbar_arrive(empty);  // this warp's wgmma reads of the A buffer have retired
    tc_epilogue<float, NCH, false, false>(pc, chunks, stg, acc, tile, wg, w4, lane);
}

template <int NCH1, int NL>
__global__ void __launch_bounds__(NTHREADS, 1) radial_embed_fwd_kernel(const __grid_constant__ RadialEmbedParams q) {
    constexpr int H = 32 * NCH1;
    constexpr int A_HALF = BM * H * 2;          // one bf16 image of a [128][H] tile
    constexpr int PQ_LD = RADJ_NB * H + 4;      // floats between the PQ blocks of consecutive type pairs
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // warp-uniform role index
    // plan: W_fold (hi, lo) | A tiles [2] (hi, lo) | epilogue staging | PQ | barriers | chunk tables
    uint8_t* sW = smem;
    uint8_t* sA = sW + 2 * q.w_half;
    float* sEpi = reinterpret_cast<float*>(sA + 2 * 2 * A_HALF);
    float* sPQ = sEpi + EPI_BYTES / 4;
    const int npair = q.num_types * q.num_types;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sPQ + ((npair * PQ_LD + 3) & ~3));  // full[2], empty[2]
    ChunkInfo* sChunk = reinterpret_cast<ChunkInfo*>(bars + 4);                     // REMB_MAX_CHUNKS x MAX_CHUNK
    const uint32_t bar0 = smem_u32(bars);
    auto full_bar = [&](int b) { return bar0 + 8u * b; };
    auto empty_bar = [&](int b) { return bar0 + 8u * (2 + b); };

    // ---- one-time setup ----
    if (threadIdx.x == 0) {
        for (int b = 0; b < 2; ++b) {
            mbar_init(full_bar(b), NPROD * 32);
            mbar_init(empty_bar(b), NCONS);
        }
        fence_barrier_init();
    }
    if (threadIdx.x >= 32 && threadIdx.x < 32 + REMB_MAX_CHUNKS * MAX_CHUNK) {
        const int i = threadIdx.x - 32, c = i / MAX_CHUNK;
        sChunk[i] = c < q.n_chunks ? tc_chunk_info<float>(q.s[c], (i % MAX_CHUNK) * 32) : ChunkInfo{nullptr, nullptr, 0, 0, 0};
    }
    for (int e = threadIdx.x; e < npair * RADJ_NB * H; e += NTHREADS) sPQ[(e / (RADJ_NB * H)) * PQ_LD + e % (RADJ_NB * H)] = __ldg(q.PQ + e);
    stage_w(sW, q.W, reinterpret_cast<const uint8_t*>(q.W) + q.w_half, q.w_half);
    fence_proxy_async();
    __syncthreads();

    if (warp < NPROD) {
        // =============================== generators ===============================
        const int rloc = warp * 16 + (lane & 15), half = lane >> 4;
        constexpr int ITEMS = H / 16;  // core-matrix columns of this thread's half row
        auto row = [&](int64_t tile) {
            const int64_t m = tile * BM + rloc;
            return m < q.M ? m : q.M - 1;  // rows beyond M compute on row M - 1; their results are never stored
        };
        int nc = 0, nn = 0;
        float v[3] = {0.f, 0.f, 0.f};
        auto fetch = [&](int64_t tile) {
            if (tile < q.num_tiles) {
                const int64_t m = row(tile);
                nc = __ldg(q.ctr + m);
                nn = __ldg(q.nbr + m);
                v[0] = __ldg(q.vec + m * 3); v[1] = __ldg(q.vec + m * 3 + 1); v[2] = __ldg(q.vec + m * 3 + 2);
            }
        };
        fetch(blockIdx.x);
        int it = 0;
        for (int64_t tile = blockIdx.x; tile < q.num_tiles; tile += gridDim.x, ++it) {
            const int pair = __ldg(q.types + nc) * q.num_types + __ldg(q.types + nn);
            const float vx = v[0], vy = v[1], vz = v[2];
            fetch(tile + gridDim.x);
            const float r = sqrtf(vx * vx + vy * vy + vz * vz);
            float B[RADJ_NB];
            bessel_basis<float, false>(r / __ldg(q.rmax_table + pair), q.p, RADJ_NB, q.bw, B, nullptr);
            const float* m = sPQ + pair * PQ_LD;
            const int buf = it & 1;
            mbar_wait(empty_bar(buf), ((it >> 1) & 1) ^ 1);
            uint8_t* st = sA + buf * 2 * A_HALF + (rloc >> 3) * (H / 8) * 128 + (rloc & 7) * 16;
#pragma unroll
            for (int i = 0; i < ITEMS; ++i) {
                const int c8 = half * ITEMS + i;
                float h[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) h[j] = 0.f;
#pragma unroll
                for (int n = 0; n < RADJ_NB; ++n) {
                    const float4 a = *reinterpret_cast<const float4*>(m + n * H + c8 * 8);
                    const float4 b = *reinterpret_cast<const float4*>(m + n * H + c8 * 8 + 4);
                    h[0] = fmaf(B[n], a.x, h[0]); h[1] = fmaf(B[n], a.y, h[1]); h[2] = fmaf(B[n], a.z, h[2]); h[3] = fmaf(B[n], a.w, h[3]);
                    h[4] = fmaf(B[n], b.x, h[4]); h[5] = fmaf(B[n], b.y, h[5]); h[6] = fmaf(B[n], b.z, h[6]); h[7] = fmaf(B[n], b.w, h[7]);
                }
                uint32_t hi[4], lo[4];
#pragma unroll
                for (int t = 0; t < 4; ++t) split_bf16x2(act_fast<NL>(h[2 * t]), act_fast<NL>(h[2 * t + 1]), hi[t], lo[t]);
                *reinterpret_cast<uint4*>(st + c8 * 128) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                *reinterpret_cast<uint4*>(st + A_HALF + c8 * 128) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
            }
            fence_proxy_async();  // generic-proxy writes, read by wgmma through the async proxy
            mbar_arrive(full_bar(buf));
        }
        return;
    }
    // =============================== consumers ===============================
    const int cw = warp - NPROD, wg = cw >> 2, w4 = cw & 3;
    float* stg = sEpi + cw * 16 * EPI_LD;
    const uint32_t sA_u = smem_u32(sA), sW_u = smem_u32(sW);
    int it = 0;
    for (int64_t tile = blockIdx.x; tile < q.num_tiles; tile += gridDim.x, ++it) {
        const int buf = it & 1;
        mbar_wait(full_bar(buf), (it >> 1) & 1);
        const uint32_t a_u = sA_u + buf * 2 * A_HALF + wg * 64 * H * 2;  // this warpgroup's 64 rows
#pragma unroll 1
        for (int c = 0; c < q.n_chunks; ++c) {
            const TcParams& pc = q.s[c];
            const ChunkInfo* ch = sChunk + c * MAX_CHUNK;
            const uint32_t w_u = sW_u + (uint32_t)q.n0[c] * H * 2;
            const bool last = c == q.n_chunks - 1;
            switch (pc.Npad / 32) {
                case 1: radial_embed_chunk<1>(pc, ch, stg, a_u, A_HALF, H, w_u, q.w_half, last, empty_bar(buf), tile, wg, w4, lane); break;
                case 2: radial_embed_chunk<2>(pc, ch, stg, a_u, A_HALF, H, w_u, q.w_half, last, empty_bar(buf), tile, wg, w4, lane); break;
                case 3: radial_embed_chunk<3>(pc, ch, stg, a_u, A_HALF, H, w_u, q.w_half, last, empty_bar(buf), tile, wg, w4, lane); break;
                default: radial_embed_chunk<4>(pc, ch, stg, a_u, A_HALF, H, w_u, q.w_half, last, empty_bar(buf), tile, wg, w4, lane); break;
            }
        }
    }
}

// =========================================================================================
// Two-layer SiLU MLP in one kernel (ab2_mlp2).  Stage 1 is the TMA-fed GEMM of linear_tma_kernel (A @ W1, converter
// warps unchanged); stage 2 multiplies the hidden layer, kept on chip, by W2.  Per 128-row tile each consumer warpgroup,
// for its own 64 rows:
//   stage 1   acc = A @ W1 from the ring (rank-1 backward: acc = gout[m] * w1[j] in fp32, no ring);
//   between   forward: pre = acc goes to HBM through the epilogue, h = silu(acc); backward: h = acc * silu'(pre).  h is
//             split into bf16 hi + lo and written to the warpgroup's resident 64 x H tile (canonical K-major), then
//             fence.proxy.async and a named barrier over the warpgroup's 128 threads.  In the backward, pre is brought in
//             by cp.async while stage 1 runs, each thread's two pre values into the very hi / lo bytes of the tile that
//             the thread later overwrites with its own result: no registers held over the main loop, no extra barrier;
//   stage 2   per column chunk of at most 64: acc2 = h @ W2[:, chunk] from the resident tile, then the epilogue into the
//             chunk's output segments.
// W1 and W2 (hi + lo) stay resident.  The hidden layer never goes to HBM, and A is read once however wide the output.
// The k16 steps, the split products and the SiLU / silu' arithmetic are those of the two ab2_linear launches it
// replaces, so the results are bitwise theirs (the rank-1 stage 1 is an exact fp32 product instead of a split MMA).
// =========================================================================================
constexpr int MLP2_MAX_H = 64;      // wider hidden layers need more than 128 registers per consumer thread (spills)
constexpr int MLP2_CHUNK = 64;      // stage-2 columns per chunk: the accumulator of stage 2 stays at 32 registers
constexpr int MLP2_MAX_CHUNKS = 4;  // N <= 256
constexpr int MLP2_TAIL = TAIL_BARS + (1 + MLP2_MAX_CHUNKS) * TAIL_CHUNK + (MAX_K / 32) * 16 + 8 * 8;

struct Mlp2Params {
    TcParams s1;                    // stage 1: A segments, K, N = Npad = H, W1 images; forward: o = {pre}
    TcParams s2[MLP2_MAX_CHUNKS];   // stage-2 column chunks: K = H, N, Npad, the chunk's output segments
    int n0[MLP2_MAX_CHUNKS];        // first column of each chunk
    int n2;                         // number of chunks
    int w2_npad;                    // columns of the whole (padded) W2 image
    int backward;
    const float* pre;               // backward: silu' argument [M][H]
    int64_t pre_ld;
    const float* gout1;             // rank-1 backward: the single Gout column (row stride gout1_ld); null otherwise
    int64_t gout1_ld;
    const float* w1row;             // rank-1 backward: the H entries of the 1 x H first matrix
};

// stage 2 of one column chunk: acc = h (resident) @ W2 chunk, epilogue into the chunk's output segments
template <int NCH>
__device__ __forceinline__ void mlp2_stage2(const TcParams& p2, const ChunkInfo* chunks, float* stg, uint32_t h_u, uint32_t h_half, int H, uint32_t w_u,
                                            uint32_t w_half, int64_t tile, int wg, int w4, int lane) {
    float acc[16 * NCH];
    tc_mma_resident<NCH>(acc, h_u, h_half, H, w_u, w_half);
    tc_epilogue<float, NCH, false>(p2, chunks, stg, acc, tile, wg, w4, lane);
}

template <int NCH1, int NL>
__global__ void __launch_bounds__(NTHREADS, 1) mlp2_kernel(const __grid_constant__ Mlp2Params q, const __grid_constant__ TmaMaps maps, int NR) {
    constexpr int G = 2, WPG = NPROD / G;
    constexpr int H = 32 * NCH1;
    const TcParams& p = q.s1;
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // warp-uniform role index
    const bool rank1 = q.gout1 != nullptr;
    const int w1_half = rank1 ? 0 : H * p.K * 2;
    const int w2_half = q.w2_npad * H * 2;
    const int stage_bytes = 2 * STAGE_HALF;
    constexpr int h_half = 64 * H * 2;  // one warpgroup's hidden tile, hi or lo image
    // plan: raw ring (1024-byte aligned) | W1 | W2 | canonical ring | hidden tiles (2 warpgroups x hi, lo) | epilogue staging | tail
    uint8_t* sRaw = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);
    uint8_t* sW1 = sRaw + (size_t)NR * TMA_BOX_BYTES;
    uint8_t* sW2 = sW1 + 2 * w1_half;
    uint8_t* sA = sW2 + 2 * w2_half;
    uint8_t* sH = sA + p.nstage * stage_bytes;
    float* sEpi = reinterpret_cast<float*>(sH + 4 * h_half);
    uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sEpi) + EPI_BYTES);
    // chunk tables: stage 1 (pre), then one per stage-2 chunk, MAX_CHUNK entries each
    ChunkInfo* sChunk = reinterpret_cast<ChunkInfo*>(reinterpret_cast<uint8_t*>(bars) + TAIL_BARS);
    int4* sKseg = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(sChunk) + (1 + MLP2_MAX_CHUNKS) * TAIL_CHUNK);
    uint64_t* rbars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(sKseg) + (MAX_K / 32) * 16);
    const uint32_t bar0 = smem_u32(bars), rbar0 = smem_u32(rbars);
    const int nkb = p.K / KC;

    // ---- one-time setup ----
    if (threadIdx.x == 0) tma_init_bars(bar0, rbar0, WPG);
    if (threadIdx.x < MAX_K / 32) {
        sKseg[threadIdx.x] = tma_kseg_entry(p, threadIdx.x);
    } else if (threadIdx.x >= 64 && threadIdx.x < 64 + (1 + MLP2_MAX_CHUNKS) * MAX_CHUNK) {
        const int i = threadIdx.x - 64, t = i / MAX_CHUNK, c0 = (i % MAX_CHUNK) * 32;
        ChunkInfo ci{nullptr, nullptr, 0, 0, 0};
        if (t == 0) ci = tc_chunk_info<float>(p, c0);
        else if (t - 1 < q.n2) ci = tc_chunk_info<float>(q.s2[t - 1], c0);
        sChunk[i] = ci;
    }
    if (!rank1) stage_w(sW1, p.Wpacked, p.Wlo, w1_half);
    stage_w(sW2, q.s2[0].Wpacked, q.s2[0].Wlo, w2_half);
    fence_proxy_async();
    __syncthreads();
    TcCtx ctx;
    ctx.sW = sW1; ctx.sA = sA; ctx.sEpi = sEpi; ctx.sChunk = sChunk; ctx.bar0 = bar0;
    ctx.nkb = nkb; ctx.stage_bytes = stage_bytes; ctx.w_half = w1_half;

    if (warp < NPROD) {
        if (!rank1) {
            const int64_t my_tiles = (p.num_tiles > blockIdx.x) ? (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
            // stage 1 loads A as it is (p.act == AB2_ACT_NONE): the converters take no nonlinearity
            tma_converter_role<G, AB2_NL_SILU>(p, maps, NR, ctx, sRaw, sKseg, rbar0, my_tiles * nkb, warp, lane);
        }
        return;
    }
    // =============================== consumers ===============================
    const int cw = warp - NPROD, wg = cw >> 2, w4 = cw & 3;
    float* stg = sEpi + cw * 16 * EPI_LD;
    uint8_t* hid = sH + wg * 2 * h_half;  // this warpgroup's hidden tile: hi, then lo
    const uint32_t hid_u = smem_u32(hid);
    const int r8 = lane >> 2, cq = 2 * (lane & 3);  // fragment: rows 16 w4 + r8 (+ 8), columns 8 j + cq (+ 1)
    const uint32_t wg_bar = 8 + wg;                 // named barrier of this warpgroup (ids 1..G are the converter groups')
    int stage = 0;
    uint32_t phase = 0;
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        // canonical K-major: byte offset of (row, k) = ((row / 8) (H / 8) + k / 8) 128 + (row % 8) 16 + (k % 8) 2
        const uint32_t off_a = (uint32_t)(threadIdx.x & 96) * (H / 8) * 8 + r8 * 16 + cq * 2, off_b = off_a + (H / 8) * 128;
        // fragment rows (rows beyond M read row M - 1: their results are never stored)
        const int64_t m0 = tile * BM + wg * 64 + w4 * 16 + r8;
        const int64_t ma = m0 < p.M ? m0 : p.M - 1, mb = m0 + 8 < p.M ? m0 + 8 : p.M - 1;
        // every warp of the warpgroup is done with the previous tile's stage-2 reads of the hidden tile
        asm volatile("bar.sync %0, %1;" ::"r"(wg_bar), "r"(128) : "memory");
        if (q.backward) {  // pre (r, c) -> hi slot of (r, c..c+1), pre (r, c + 1) -> its lo slot
            const float* ra = q.pre + ma * q.pre_ld + cq;
            const float* rb = q.pre + mb * q.pre_ld + cq;
#pragma unroll
            for (int j = 0; j < 4 * NCH1; ++j) {
                cp_async4(hid_u + off_a + j * 128, ra + 8 * j);
                cp_async4(hid_u + h_half + off_a + j * 128, ra + 8 * j + 1);
                cp_async4(hid_u + off_b + j * 128, rb + 8 * j);
                cp_async4(hid_u + h_half + off_b + j * 128, rb + 8 * j + 1);
            }
            cp_async_commit();
        }
        // hidden value i = 4 j + e of this thread's fragment -> bf16 hi + lo in the tile.  In the backward the slot still
        // holds pre (see above) and is read just before it is overwritten.  (Values are formed on the way to shared
        // memory: registers an MMA accumulates into are never written by other instructions, which would make ptxas
        // serialise the wgmma pipeline.)
        auto slot = [&](int i) { return hid + ((i & 2) ? off_b : off_a) + (i >> 2) * 128 + ((i & 1) ? h_half : 0); };
        auto pre_at = [&](int i) { return *reinterpret_cast<const float*>(slot(i)); };
        auto store_hidden = [&](auto&& h) {
#pragma unroll
            for (int j = 0; j < 4 * NCH1; ++j) {
                const float h0 = h(4 * j), h1 = h(4 * j + 1), h2 = h(4 * j + 2), h3 = h(4 * j + 3);
                uint32_t hi, lo;
                split_bf16x2(h0, h1, hi, lo);
                *reinterpret_cast<uint32_t*>(slot(4 * j)) = hi;
                *reinterpret_cast<uint32_t*>(slot(4 * j + 1)) = lo;
                split_bf16x2(h2, h3, hi, lo);
                *reinterpret_cast<uint32_t*>(slot(4 * j + 2)) = hi;
                *reinterpret_cast<uint32_t*>(slot(4 * j + 3)) = lo;
            }
        };
        if (rank1) {
            const float ga = __ldg(q.gout1 + ma * q.gout1_ld), gb = __ldg(q.gout1 + mb * q.gout1_ld);
            cp_async_wait<0>();  // this thread's own copies: visible to it once complete
            store_hidden([&](int i) {
                const float w = __ldg(q.w1row + 8 * (i >> 2) + cq + (i & 1));
                return ((i & 2) ? gb : ga) * w * dact_fast<NL>(pre_at(i));
            });
        } else {
            float acc[16 * NCH1];
            tc_mma_ring<true, NCH1>(acc, p, ctx, wg, lane, stage, phase);
            if (!q.backward) {
                tc_epilogue<float, NCH1, false>(p, sChunk, stg, acc, tile, wg, w4, lane);  // pre
                store_hidden([&](int i) { return act_fast<NL>(acc[i]); });
            } else {
                cp_async_wait<0>();
                store_hidden([&](int i) { return acc[i] * dact_fast<NL>(pre_at(i)); });
            }
        }
        fence_proxy_async();  // generic-proxy writes, read by wgmma through the async proxy
        asm volatile("bar.sync %0, %1;" ::"r"(wg_bar), "r"(128) : "memory");
#pragma unroll 1
        for (int c = 0; c < q.n2; ++c) {
            const TcParams& p2 = q.s2[c];
            const ChunkInfo* ch = sChunk + (1 + c) * MAX_CHUNK;
            const uint32_t w_u = smem_u32(sW2) + (uint32_t)q.n0[c] * H * 2;
            if (p2.Npad == 32) mlp2_stage2<1>(p2, ch, stg, hid_u, h_half, H, w_u, w2_half, tile, wg, w4, lane);
            else mlp2_stage2<2>(p2, ch, stg, hid_u, h_half, H, w_u, w2_half, tile, wg, w4, lane);
        }
    }
}

// =========================================================================================
// Last latent MLP + readout MLP in one kernel (ab2_mlp2_readout).  The readout reads X[:, :P + S] = [X[:, :P] | x_L]
// and the last latent MLP reads [X[:, :P] | s] and writes x_L = X[:, P:P+S], so one kernel streams X[:, :P] once and
// keeps x_L (forward) and its gradient (backward) on chip.  W1_ro = [W1_ro_a ; W1_ro_b] split by rows at P; w2_ro is
// the readout's H x 1 output layer (fp32).  H = S = 64.  Per 128-row tile each consumer warpgroup, for its own 64 rows:
//   forward   ring over A = [X[:, :P] | s]: acc = A @ W1_lat and, over the first P columns only, acc_r = A @ W1_ro_a;
//             pre_L = acc to HBM; h = silu(acc) to the on-chip tile T; x = h @ W2_lat to HBM (x_L) and, split into
//             bf16 hi + lo as the converters split it, to T; acc_r += x @ W1_ro_b, which continues the readout's k16
//             order over K = P + S, so pre_r = acc_r is bitwise the readout's; pre_r to HBM;
//             Ez = sum_j silu(pre_r[j]) w2_ro[j] in fp32 (a quad shuffle; the readout MMA's split-bf16 w2_ro is
//             replaced by the exact fp32 product).
//   backward  g_r = gEz w2_ro silu'(pre_r) in fp32 (the rank-1 stage of mlp2_kernel) to T_r; g_x = g_r @ W1_ro^T[:, P:]
//             to T_x (never to HBM); g_h = (g_x @ W2_lat^T) silu'(pre_L) to T_h; then per column chunk (<= 64) of
//             [gX[:, :P] | gs]: T_h @ W1_lat^T[:, chunk] (+ T_r @ W1_ro^T[:, chunk] for the gX chunks, added once in
//             fp32: the readout's gX written and then accumulated into, without the round trip).  pre_r and pre_L
//             arrive by cp.async as in mlp2_kernel.  No ring: the converter warps only stage the weights.
// Everything other than Ez is bitwise the two mlp2_kernel launches it replaces.
// =========================================================================================
constexpr int RO_H = 64;                    // hidden width of both MLPs and the width S of x_L
constexpr int RO_TILE = 64 * RO_H * 2;      // one warpgroup's 64 x 64 on-chip operand, hi or lo image (8 KB)
constexpr int RO_MAX_CHUNKS = 4;            // backward output chunks: P + U <= 256
constexpr int RO_TAIL = TAIL_BARS + RO_MAX_CHUNKS * TAIL_CHUNK + (MAX_K / 32) * 16 + 8 * 8 + RO_H * 4;

struct Mlp2RoParams {
    TcParams s1;                  // forward: ring GEMM over [X[:, :P] | s] (K = P + U, N = H) with o = {pre_L}; backward: M, num_tiles
    TcParams o[RO_MAX_CHUNKS];    // forward: {x_L, pre_r}; backward: the column chunks of [gX[:, :P] | gs]
    int n0[RO_MAX_CHUNKS];        // backward: first column of each chunk
    int n_chunks;
    int P;
    const void* w[4];             // packed images, forward: W1_lat, W2_lat, W1_ro_a, W1_ro_b; backward: W1_ro^T, W2_lat^T, W1_lat^T
    int w_half[4];                // bytes of each hi (= lo) image
    const float* w2ro;            // H fp32
    float* ez;                    // forward: Ez (written); backward: gEz (read)
    int64_t ez_ld;
    const float* pre_l;           // backward: silu' arguments
    int64_t pre_l_ld;
    const float* pre_r;
    int64_t pre_r_ld;
};

// this thread's 32 accumulator values (fragment of rows r8, r8 + 8 and columns 8 j + cq (+ 1)) -> bf16 hi + lo images of a
// warpgroup's 64 x 64 canonical K-major tile, as the converters split; h(i) gives value i
template <typename F>
__device__ __forceinline__ void ro_store_tile(uint8_t* t, uint32_t off_a, uint32_t off_b, F&& h) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        uint32_t hi, lo;
        split_bf16x2(h(4 * j), h(4 * j + 1), hi, lo);
        *reinterpret_cast<uint32_t*>(t + off_a + j * 128) = hi;
        *reinterpret_cast<uint32_t*>(t + RO_TILE + off_a + j * 128) = lo;
        split_bf16x2(h(4 * j + 2), h(4 * j + 3), hi, lo);
        *reinterpret_cast<uint32_t*>(t + off_b + j * 128) = hi;
        *reinterpret_cast<uint32_t*>(t + RO_TILE + off_b + j * 128) = lo;
    }
}

// pre (r, c) -> hi slot of (r, c..c+1), pre (r, c + 1) -> its lo slot, for this thread's fragment (see mlp2_kernel)
__device__ __forceinline__ void ro_fetch_pre(uint32_t t_u, uint32_t off_a, uint32_t off_b, const float* ra, const float* rb) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        cp_async4(t_u + off_a + j * 128, ra + 8 * j);
        cp_async4(t_u + RO_TILE + off_a + j * 128, ra + 8 * j + 1);
        cp_async4(t_u + off_b + j * 128, rb + 8 * j);
        cp_async4(t_u + RO_TILE + off_b + j * 128, rb + 8 * j + 1);
    }
    cp_async_commit();
}

__device__ __forceinline__ float ro_pre_at(const uint8_t* t, uint32_t off_a, uint32_t off_b, int i) {
    return *reinterpret_cast<const float*>(t + ((i & 2) ? off_b : off_a) + (i >> 2) * 128 + ((i & 1) ? RO_TILE : 0));
}

// shared-memory plan of mlp2_readout_fwd_kernel: raw ring (1024-byte aligned) | W1_lat | W2_lat | W1_ro_a | W1_ro_b |
// canonical ring | tiles (2 warpgroups x hi, lo) | epilogue staging | tail (barriers, chunk tables pre_L / x_L / pre_r,
// k-chunk table, raw-slot barriers, w2_ro)
struct RoFwdPlan {
    uint8_t* raw;
    uint8_t* w[4];
    uint8_t* a;
    uint8_t* t;
    float* epi;
    uint64_t* bars;
    ChunkInfo* chunk;
    int4* kseg;
    uint64_t* rbars;
    float* w2ro;
    __device__ __forceinline__ RoFwdPlan(uint8_t* smem, const Mlp2RoParams& q, int NR) {
        raw = smem + ((1024u - (smem_u32(smem) & 1023u)) & 1023u);
        w[0] = raw + (size_t)NR * TMA_BOX_BYTES;
#pragma unroll
        for (int i = 1; i < 4; ++i) w[i] = w[i - 1] + 2 * q.w_half[i - 1];
        a = w[3] + 2 * q.w_half[3];
        t = a + q.s1.nstage * 2 * STAGE_HALF;
        epi = reinterpret_cast<float*>(t + 4 * RO_TILE);
        bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(epi) + EPI_BYTES);
        chunk = reinterpret_cast<ChunkInfo*>(reinterpret_cast<uint8_t*>(bars) + TAIL_BARS);
        kseg = reinterpret_cast<int4*>(reinterpret_cast<uint8_t*>(chunk) + RO_MAX_CHUNKS * TAIL_CHUNK);
        rbars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(kseg) + (MAX_K / 32) * 16);
        w2ro = reinterpret_cast<float*>(rbars + 8);
    }
    __device__ __forceinline__ TcCtx ctx(const Mlp2RoParams& q) const {
        TcCtx c;
        c.sW = w[0]; c.sA = a; c.sEpi = epi; c.sChunk = chunk; c.bar0 = smem_u32(bars);
        c.nkb = q.s1.K / KC; c.stage_bytes = 2 * STAGE_HALF; c.w_half = q.w_half[0];
        return c;
    }
};

template <int NL>
__global__ void __launch_bounds__(NTHREADS, 1) mlp2_readout_fwd_kernel(const __grid_constant__ Mlp2RoParams q, const __grid_constant__ TmaMaps maps,
                                                                        int NR) {
    constexpr int G = 2, WPG = NPROD / G;
    const TcParams& p = q.s1;
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);  // warp-uniform role index

    // ---- one-time setup ----
    {
        const RoFwdPlan sp(smem, q, NR);
        if (threadIdx.x == 0) tma_init_bars(smem_u32(sp.bars), smem_u32(sp.rbars), WPG);
        if (threadIdx.x < MAX_K / 32) {
            sp.kseg[threadIdx.x] = tma_kseg_entry(p, threadIdx.x);
        } else if (threadIdx.x >= 64 && threadIdx.x < 64 + 3 * MAX_CHUNK) {
            const int i = threadIdx.x - 64, t = i / MAX_CHUNK, c0 = (i % MAX_CHUNK) * 32;
            sp.chunk[i] = tc_chunk_info<float>(t == 0 ? p : q.o[t - 1], c0);
        } else if (threadIdx.x >= 128 && threadIdx.x < 128 + RO_H) {
            sp.w2ro[threadIdx.x - 128] = q.w2ro[threadIdx.x - 128];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) stage_w(sp.w[i], q.w[i], reinterpret_cast<const uint8_t*>(q.w[i]) + q.w_half[i], q.w_half[i]);
        fence_proxy_async();
        __syncthreads();
        if (warp < NPROD) {
            const int64_t my_tiles = (p.num_tiles > blockIdx.x) ? (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
            // the ring carries A as it is (p.act == AB2_ACT_NONE): the converters take no nonlinearity
            tma_converter_role<G, AB2_NL_SILU>(p, maps, NR, sp.ctx(q), sp.raw, sp.kseg, smem_u32(sp.rbars), my_tiles * (p.K / KC), warp,
                                               threadIdx.x & 31);
            return;
        }
    }
    // =============================== consumers ===============================
    const int cw = warp - NPROD, wg = cw >> 2, w4 = cw & 3;
    const uint32_t wg_bar = 8 + wg;  // named barrier of this warpgroup (ids 1..G are the converter groups')
    const int nkb_r = q.P / KC;
    auto wg_sync = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(wg_bar), "r"(128) : "memory"); };
    int stage = 0;
    uint32_t phase = 0;
    const RoFwdPlan sp(smem, q, NR);
    const TcCtx ctx = sp.ctx(q);
    float* stg = sp.epi + cw * 16 * EPI_LD;
    uint8_t* tl = sp.t + wg * 2 * RO_TILE;  // this warpgroup's tile: hi, then lo
    const uint32_t tl_u = smem_u32(tl);
    const uint32_t wa_u = smem_u32(sp.w[2]), wa_half = q.w_half[2], wa_sbo = (uint32_t)(q.P / 8) * 128;
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        // The lane index is re-read per tile: the lane-dependent addresses of the three epilogues are then formed inside
        // the loop.  Hoisted out of it they stay live next to the 64 accumulator registers of the ring and spill.
        int lane;
        asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
        const int r8 = lane >> 2, cq = 2 * (lane & 3);  // fragment: rows 16 w4 + r8 (+ 8), columns 8 j + cq (+ 1)
        // canonical K-major: byte offset of (row, k) = ((row / 8) (H / 8) + k / 8) 128 + (row % 8) 16 + (k % 8) 2
        const uint32_t off_a = (uint32_t)w4 * 32 * (RO_H / 8) * 8 + r8 * 16 + cq * 2, off_b = off_a + (RO_H / 8) * 128;
        wg_sync();  // every warp of the warpgroup is done with the previous tile's reads of T
        float acc[32], acc_r[32];
        // acc_r = X[:, :P] @ W1_ro_a from the same ring stages, with the products in the order of the readout's ring
        tc_mma_ring<true, 2>(acc, p, ctx, wg, lane, stage, phase, [&](int kb, int ks, uint64_t da_hi, uint64_t da_lo) {
            if (kb < nkb_r) {
                const uint32_t wk = wa_u + (uint32_t)(kb * (KC / 8) + ks * 2) * 128;
                const uint64_t db_hi = make_desc(wk, 128, wa_sbo), db_lo = make_desc(wk + wa_half, 128, wa_sbo);
                wgmma_bf16<2>(acc_r, da_hi, db_hi, (kb | ks) ? 1u : 0u);
                wgmma_bf16<2>(acc_r, da_lo, db_hi, 1u);
                wgmma_bf16<2>(acc_r, da_hi, db_lo, 1u);
            }
        });
        tc_epilogue<float, 2, false, false>(p, sp.chunk, stg, acc, tile, wg, w4, lane);  // pre_L
        ro_store_tile(tl, off_a, off_b, [&](int i) { return act_fast<NL>(acc[i]); });
        fence_proxy_async();  // generic-proxy writes, read by wgmma through the async proxy
        wg_sync();
        {
            float x[32];
            tc_mma_resident<2>(x, tl_u, RO_TILE, RO_H, smem_u32(sp.w[1]), q.w_half[1]);
            wg_sync();  // every warp's wgmma reads of h have completed before T is overwritten
            tc_epilogue<float, 2, false, false>(q.o[0], sp.chunk + MAX_CHUNK, stg, x, tile, wg, w4, lane);  // x_L
            ro_store_tile(tl, off_a, off_b, [&](int i) { return x[i]; });
        }
        fence_proxy_async();
        wg_sync();
        tc_mma_resident<2>(acc_r, tl_u, RO_TILE, RO_H, smem_u32(sp.w[3]), q.w_half[3], /*accumulate=*/true);
        tc_epilogue<float, 2, false, false>(q.o[1], sp.chunk + 2 * MAX_CHUNK, stg, acc_r, tile, wg, w4, lane);  // pre_r
        // Ez: this thread's 16 columns of rows r8 and r8 + 8, then the sum over the 4 lanes of the quad
        float ea = 0.f, eb = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float2 w = *reinterpret_cast<const float2*>(sp.w2ro + 8 * j + cq);
            ea = fmaf(act_fast<NL>(acc_r[4 * j]), w.x, ea);
            ea = fmaf(act_fast<NL>(acc_r[4 * j + 1]), w.y, ea);
            eb = fmaf(act_fast<NL>(acc_r[4 * j + 2]), w.x, eb);
            eb = fmaf(act_fast<NL>(acc_r[4 * j + 3]), w.y, eb);
        }
        ea += __shfl_xor_sync(0xffffffffu, ea, 1);
        eb += __shfl_xor_sync(0xffffffffu, eb, 1);
        ea += __shfl_xor_sync(0xffffffffu, ea, 2);
        eb += __shfl_xor_sync(0xffffffffu, eb, 2);
        const int64_t m0 = tile * BM + wg * 64 + w4 * 16 + r8;
        if ((lane & 3) == 0) {
            if (m0 < p.M) q.ez[m0 * q.ez_ld] = ea;
            if (m0 + 8 < p.M) q.ez[(m0 + 8) * q.ez_ld] = eb;
        }
    }
}

// backward output chunk c: acc = T_h @ W1_lat^T[:, chunk] (+ T_r @ W1_ro^T[:, chunk]), epilogue into the chunk's output
template <int NCH>
__device__ __forceinline__ void ro_bwd_chunk(const TcParams& pc, const ChunkInfo* chunks, float* stg, uint32_t th_u, uint32_t wl_u, uint32_t wl_half,
                                             uint32_t tr_u, uint32_t wr_u, uint32_t wr_half, bool with_ro, int64_t tile, int wg, int w4, int lane) {
    float acc[16 * NCH];
    tc_mma_resident<NCH>(acc, th_u, RO_TILE, RO_H, wl_u, wl_half);
    if (with_ro) {
        float acc2[16 * NCH], sum[16 * NCH];
        tc_mma_resident<NCH>(acc2, tr_u, RO_TILE, RO_H, wr_u, wr_half);
#pragma unroll
        for (int i = 0; i < 16 * NCH; ++i) sum[i] = acc[i] + acc2[i];
        tc_epilogue<float, NCH, false>(pc, chunks, stg, sum, tile, wg, w4, lane);
    } else {
        tc_epilogue<float, NCH, false>(pc, chunks, stg, acc, tile, wg, w4, lane);
    }
}

template <int NL>
__global__ void __launch_bounds__(NTHREADS, 1) mlp2_readout_bwd_kernel(const __grid_constant__ Mlp2RoParams q) {
    const TcParams& p = q.s1;
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;  // warp-uniform role index
    // plan: W1_ro^T | W2_lat^T | W1_lat^T | tiles T_r, T_x, T_h (2 warpgroups x hi, lo each) | epilogue staging | tail
    uint8_t* sWi[3];
    sWi[0] = smem;
    for (int i = 1; i < 3; ++i) sWi[i] = sWi[i - 1] + 2 * q.w_half[i - 1];
    uint8_t* sT = sWi[2] + 2 * q.w_half[2];
    float* sEpi = reinterpret_cast<float*>(sT + 3 * 4 * RO_TILE);
    ChunkInfo* sChunk = reinterpret_cast<ChunkInfo*>(reinterpret_cast<uint8_t*>(sEpi) + EPI_BYTES + TAIL_BARS);
    if (threadIdx.x < RO_MAX_CHUNKS * MAX_CHUNK) {
        const int t = threadIdx.x / MAX_CHUNK;
        ChunkInfo ci{nullptr, nullptr, 0, 0, 0};
        if (t < q.n_chunks) ci = tc_chunk_info<float>(q.o[t], (threadIdx.x % MAX_CHUNK) * 32);
        sChunk[threadIdx.x] = ci;
    }
    for (int i = 0; i < 3; ++i) stage_w(sWi[i], q.w[i], reinterpret_cast<const uint8_t*>(q.w[i]) + q.w_half[i], q.w_half[i]);
    fence_proxy_async();
    __syncthreads();
    if (warp < NPROD) return;
    // =============================== consumers ===============================
    const int cw = warp - NPROD, wg = cw >> 2, w4 = cw & 3;
    float* stg = sEpi + cw * 16 * EPI_LD;
    uint8_t* t_r = sT + wg * 2 * RO_TILE;  // this warpgroup's tiles (hi, then lo): T_r, T_x, T_h
    uint8_t* t_x = t_r + 4 * RO_TILE;
    uint8_t* t_h = t_x + 4 * RO_TILE;
    const uint32_t tr_u = smem_u32(t_r), tx_u = smem_u32(t_x), th_u = smem_u32(t_h);
    const uint32_t wr_u = smem_u32(sWi[0]), wl_u = smem_u32(sWi[2]);
    const int r8 = lane >> 2, cq = 2 * (lane & 3);
    const uint32_t wg_bar = 8 + wg;
    const uint32_t off_a = (uint32_t)(threadIdx.x & 96) * (RO_H / 8) * 8 + r8 * 16 + cq * 2, off_b = off_a + (RO_H / 8) * 128;
    auto wg_sync = [&]() { asm volatile("bar.sync %0, %1;" ::"r"(wg_bar), "r"(128) : "memory"); };
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int64_t m0 = tile * BM + wg * 64 + w4 * 16 + r8;  // rows beyond M read row M - 1: their results are never stored
        const int64_t ma = m0 < p.M ? m0 : p.M - 1, mb = m0 + 8 < p.M ? m0 + 8 : p.M - 1;
        wg_sync();  // every warp of the warpgroup is done with the previous tile's reads of T_r, T_x, T_h
        ro_fetch_pre(tr_u, off_a, off_b, q.pre_r + ma * q.pre_r_ld + cq, q.pre_r + mb * q.pre_r_ld + cq);
        ro_fetch_pre(th_u, off_a, off_b, q.pre_l + ma * q.pre_l_ld + cq, q.pre_l + mb * q.pre_l_ld + cq);
        const float ga = __ldg(q.ez + ma * q.ez_ld), gb = __ldg(q.ez + mb * q.ez_ld);
        cp_async_wait<1>();  // pre_r (this thread's own copies: visible to it once complete)
        ro_store_tile(t_r, off_a, off_b, [&](int i) {
            const float w = __ldg(q.w2ro + 8 * (i >> 2) + cq + (i & 1));
            return ((i & 2) ? gb : ga) * w * dact_fast<NL>(ro_pre_at(t_r, off_a, off_b, i));
        });
        fence_proxy_async();
        wg_sync();
        {
            float gx[32];  // g_x = g_r @ W1_ro^T[:, P:P+S]
            tc_mma_resident<2>(gx, tr_u, RO_TILE, RO_H, wr_u + (uint32_t)q.P * RO_H * 2, q.w_half[0]);
            ro_store_tile(t_x, off_a, off_b, [&](int i) { return gx[i]; });
        }
        fence_proxy_async();
        wg_sync();
        {
            float gh[32];  // g_h = (g_x @ W2_lat^T) silu'(pre_L)
            tc_mma_resident<2>(gh, tx_u, RO_TILE, RO_H, smem_u32(sWi[1]), q.w_half[1]);
            cp_async_wait<0>();
            ro_store_tile(t_h, off_a, off_b, [&](int i) { return gh[i] * dact_fast<NL>(ro_pre_at(t_h, off_a, off_b, i)); });
        }
        fence_proxy_async();
        wg_sync();
#pragma unroll 1
        for (int c = 0; c < q.n_chunks; ++c) {
            const TcParams& pc = q.o[c];
            const uint32_t n0 = (uint32_t)q.n0[c];
            const bool with_ro = (int)n0 < q.P;
            if (pc.Npad == 32)
                ro_bwd_chunk<1>(pc, sChunk + c * MAX_CHUNK, stg, th_u, wl_u + n0 * RO_H * 2, q.w_half[2], tr_u, wr_u + n0 * RO_H * 2, q.w_half[0],
                                with_ro, tile, wg, w4, lane);
            else
                ro_bwd_chunk<2>(pc, sChunk + c * MAX_CHUNK, stg, th_u, wl_u + n0 * RO_H * 2, q.w_half[2], tr_u, wr_u + n0 * RO_H * 2, q.w_half[0],
                                with_ro, tile, wg, w4, lane);
        }
    }
}

// W[K][N] (row-major TSrc) -> canonical K-major no-swizzle bf16 images (hi, lo), Npad rows:
//   byte offset of (n, k) = ((n/8)*(K/8) + k/8)*128 + (n%8)*16 + (k%8)*2
template <typename TSrc>
__global__ void pack_w_kernel(int K, int N, int Npad, const TSrc* __restrict__ W, bf16* __restrict__ out) {
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= Npad * K) return;
    const int n = e / K, k = e % K;
    const float w = (n < N) ? to_acc<float>(W[(int64_t)k * N + n]) : 0.f;
    const bf16 h = __float2bfloat16_rn(w);
    const bf16 l = __float2bfloat16_rn(w - __bfloat162float(h));
    const int64_t off = ((int64_t)(n / 8) * (K / 8) + k / 8) * 64 + (n % 8) * 8 + (k % 8);
    out[off] = h;
    out[(int64_t)Npad * K + off] = l;
}

}  // namespace

// W images are padded to whole 32-column chunks (the wgmma N granularity used here)
static int tc_npad(int N) { return (N + 31) / 32 * 32; }

extern "C" int64_t ab2_linear_packed_bytes(int dtype, int K, int N) {
    if (dtype == AB2_F64 || K % 16 != 0 || K <= 0 || K > MAX_K || N <= 0) return 0;
    const int Npad = tc_npad(N);
    return (int64_t)Npad * K * 2 * 2;  // hi + lo images (any N: wide outputs run as column slices, see ab2_linear_tc_try)
}

// widest column slice (multiple of 32, <= MAX_N) whose resident W image fits MAX_W_BYTES
static int tc_slice_cap(int dtype, int K) {
    const int per_col = K * 2 * (dtype == AB2_F32 ? 2 : 1);
    int cap = (MAX_W_BYTES / per_col) / 32 * 32;
    if (cap > MAX_N) cap = MAX_N;
    return cap;
}

extern "C" int ab2_linear_pack(int dtype, int K, int N, const void* W, void* packed, void* stream) {
    AB2_CHECK_ARG(ab2_linear_packed_bytes(dtype, K, N) > 0, "shape not supported by the tensor-core path");
    AB2_CHECK_ARG(W && packed, "null pointer");
    const int Npad = tc_npad(N);
    cudaStream_t st = (cudaStream_t)stream;
    const int total = Npad * K;
    if (dtype == AB2_F32)
        pack_w_kernel<float><<<(total + 255) / 256, 256, 0, st>>>(K, N, Npad, (const float*)W, (bf16*)packed);
    else
        pack_w_kernel<bf16><<<(total + 255) / 256, 256, 0, st>>>(K, N, Npad, (const bf16*)W, (bf16*)packed);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// ---- host side of the TMA variant: tensor maps (driver entry point fetched through the runtime, no libcuda link) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn tc_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
        else
            cudaGetLastError();
    }
    return fn;
}

// 2-D map of one fp32 row segment: dims {width, M}, row pitch ld*4 bytes, box 32 columns x 128 rows, 128-byte swizzle
static bool tc_make_map(CUtensorMap* map, const void* ptr, int64_t ld, int width, int64_t M) {
    EncodeTiledFn fn = tc_encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)M};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    const cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)BM};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// runs f(std::integral_constant<int, NL>) for the AB2_NL_* code nonlin (validated by the caller)
template <typename F>
static int tc_with_nl(int nonlin, F&& f) {
    switch (nonlin) {
        case AB2_NL_MISH: return f(std::integral_constant<int, AB2_NL_MISH>{});
        case AB2_NL_GELU: return f(std::integral_constant<int, AB2_NL_GELU>{});
        default: return f(std::integral_constant<int, AB2_NL_SILU>{});
    }
}

static int tc_launch_tma(TcParams& p, int w_bytes, int stage_bytes, int max_smem, unsigned grid, cudaStream_t st, bool dry, int nonlin) {
    TmaMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (!tc_encode_fn()) return -1;
    for (int s = 0; s < p.n_a && !dry; ++s) {
        if (!tc_make_map(&maps.a[s], p.a[s].ptr, p.a[s].ld, p.a[s].width, p.M)) return -1;
        if (p.a[s].aux && !tc_make_map(&maps.x[s], p.a[s].aux, p.a[s].aux_ld, p.a[s].width, p.M)) return -1;
    }
    const int raw_slot = TMA_BOX_BYTES * (p.has_aux ? 2 : 1);
    // shared-memory plan (1 KB slack for the swizzle alignment): G converter groups, NR raw slots, cn canonical stages with
    // NR % G == 0 and cn % G == 0 (see the kernel); deepest pipeline that fits
    const int plans[6][3] = {{4, 8, 4}, {4, 4, 4}, {2, 4, 4}, {2, 2, 4}, {2, 4, 2}, {2, 2, 2}};  // {G, NR, cn}
    int G = 0, NR = 0, nstage = 0;
    size_t smem = 0;
    for (int q = 0; q < 6 && !G; ++q) {
        const size_t need = 1024 + ((w_bytes + 127) & ~127) + (size_t)plans[q][2] * stage_bytes + EPI_BYTES + TAIL_BYTES +
                            (size_t)plans[q][1] * raw_slot;
        if (need <= (size_t)max_smem) { G = plans[q][0]; NR = plans[q][1]; nstage = plans[q][2]; smem = need; }
    }
    if (!G) return -1;
    if (dry) return 0;
    p.nstage = nstage;
    auto go = [&](auto kern) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return -1;
        }
        kern<<<grid, NTHREADS, smem, st>>>(p, maps, NR);
        return 0;
    };
    return tc_with_nl(nonlin, [&](auto nl) -> int {
        constexpr int NL = decltype(nl)::value;
        switch ((G == 4 ? 4 : 0) + p.Npad / 32) {
            case 1: return go(linear_tma_kernel<2, 1, NL>);
            case 2: return go(linear_tma_kernel<2, 2, NL>);
            case 3: return go(linear_tma_kernel<2, 3, NL>);
            case 4: return go(linear_tma_kernel<2, 4, NL>);
            case 5: return go(linear_tma_kernel<4, 1, NL>);
            case 6: return go(linear_tma_kernel<4, 2, NL>);
            case 7: return go(linear_tma_kernel<4, 3, NL>);
            case 8: return go(linear_tma_kernel<4, 4, NL>);
        }
        return -1;
    });
}

// SM count and opt-in shared memory per block of the current device (queried once)
static void tc_device_limits(int& num_sms, int& max_smem) {
    static int sms = 0, smem = 0;
    if (sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    num_sms = sms;
    max_smem = smem;
}

// One column slice [n0, n0 + N) of the GEMM with its W images resident in shared memory.
static int tc_launch_slice(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                           const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* Whi, const void* Wlo,
                           int n_o, void* const* o_ptr, const int64_t* o_ld, const int32_t* o_width, const int32_t* o_accum, int epi,
                           const void* aux, int64_t aux_ld, cudaStream_t st, int nonlin, bool dry = false) {
    const int has_aux = (act == AB2_ACT_MUL_DSILU && a_aux) ? 1 : 0;
    if (tc_npad(N) > MAX_N) return -1;
    int num_sms = 0, max_smem = 0;
    tc_device_limits(num_sms, max_smem);
    TcParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.K = K; p.N = N; p.Npad = tc_npad(N); p.n_a = n_a; p.act = act; p.Wpacked = Whi; p.Wlo = Wlo; p.n_o = n_o;
    p.epi = epi; p.aux = aux; p.aux_ld = aux_ld; p.num_tiles = (M + BM - 1) / BM;
    for (int s = 0; s < n_a; ++s) {
        p.a[s].ptr = a_ptr[s]; p.a[s].ld = a_ld[s]; p.a[s].width = a_width[s];
        p.a[s].aux = has_aux ? a_aux[s] : nullptr; p.a[s].aux_ld = has_aux ? a_aux_ld[s] : 0;
    }
    p.has_aux = has_aux;
    for (int s = 0; s < n_o; ++s) { p.o[s].ptr = o_ptr[s]; p.o[s].ld = o_ld[s]; p.o[s].width = o_width[s]; p.o[s].accum = o_accum ? o_accum[s] : 0; }
    const bool split = dtype == AB2_F32;
    const int w_bytes = p.Npad * K * 2 * (split ? 2 : 1);
    const int stage_bytes = STAGE_HALF * (split ? 2 : 1);
    // shared-memory plan: prefer deep raw prefetch (4) and 4 canonical stages; shrink until it fits
    int nstage = 0, raw_depth = 0;
    size_t smem = 0;
    const int raw_stage = RAW_STAGE * (has_aux ? 2 : 1);
    const int plans[4][2] = {{4, NSTAGE}, {4, 2}, {2, NSTAGE}, {2, 2}};
    for (int q = 0; q < 4 && !nstage; ++q) {
        const size_t need = ((w_bytes + 127) & ~127) + (size_t)plans[q][1] * stage_bytes + (size_t)plans[q][0] * raw_stage + EPI_BYTES +
                            TAIL_BYTES;
        if ((int)need <= max_smem) { raw_depth = plans[q][0]; nstage = plans[q][1]; smem = need; }
    }
    if (!nstage) return -1;
    if (dry) return 0;
    p.nstage = nstage;
    p.raw_depth = raw_depth;
    p.debug = g_ab2_opt_tc_debug;
    const unsigned grid = (unsigned)((p.num_tiles < num_sms) ? p.num_tiles : num_sms);
    // ---- TMA-producer kernel: fp32 storage, every A segment (and K) a multiple of 32 columns ----
    bool tma_ok = g_ab2_opt_linear_tma && split && K % KC == 0 && M < ((int64_t)1 << 31);
    for (int s = 0; s < n_a && tma_ok; ++s) tma_ok = a_width[s] % KC == 0;
    if (tma_ok) {
        const int rc = tc_launch_tma(p, w_bytes, stage_bytes, max_smem, grid, st, dry, nonlin);
        if (rc == 0) return 0;
    }
    auto go = [&](auto kern) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return -1;
        }
        kern<<<grid, NTHREADS, smem, st>>>(p);
        return 0;
    };
    return tc_with_nl(nonlin, [&](auto nl) -> int {
        constexpr int NL = decltype(nl)::value;
        switch ((split ? 4 : 0) + p.Npad / 32) {
            case 1: return go(linear_tc_kernel<bf16, false, 1, NL>);
            case 2: return go(linear_tc_kernel<bf16, false, 2, NL>);
            case 3: return go(linear_tc_kernel<bf16, false, 3, NL>);
            case 4: return go(linear_tc_kernel<bf16, false, 4, NL>);
            case 5: return go(linear_tc_kernel<float, true, 1, NL>);
            case 6: return go(linear_tc_kernel<float, true, 2, NL>);
            case 7: return go(linear_tc_kernel<float, true, 3, NL>);
            case 8: return go(linear_tc_kernel<float, true, 4, NL>);
        }
        return -1;
    });
}

// returns 0 if launched, -1 if this call is not eligible (caller falls back to linear.cu).
// Outputs wider than MAX_N columns, or whose W image exceeds the shared-memory budget, run as column slices (one launch
// per slice, each with its W slice resident; the A rows are re-read per slice).
int ab2_linear_tc_try(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                      const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* Wpacked, int n_o, void* const* o_ptr, const int64_t* o_ld,
                      const int32_t* o_width, const int32_t* o_accum, int epi, const void* aux, int64_t aux_ld, cudaStream_t st, int nonlin) {
    if (!g_ab2_opt_linear_tc || !Wpacked || dtype == AB2_F64) return -1;
    if (ab2_linear_packed_bytes(dtype, K, N) == 0) return -1;
    const int esz = (dtype == AB2_F32) ? 4 : 2;
    for (int s = 0; s < n_a; ++s) {
        if (a_width[s] % 8 != 0) return -1;
        if ((reinterpret_cast<uintptr_t>(a_ptr[s]) % 16) != 0 || (a_ld[s] * esz) % 16 != 0) return -1;
        if (act == AB2_ACT_MUL_DSILU && a_aux && a_aux[s] &&
            ((reinterpret_cast<uintptr_t>(a_aux[s]) % 16) != 0 || (a_aux_ld[s] * esz) % 16 != 0)) return -1;
    }
    const int cap = tc_slice_cap(dtype, K);
    if (cap < 32) return -1;
    const int Npad_full = tc_npad(N);
    const int nslices = (N + cap - 1) / cap;
    int width = ((N + nslices - 1) / nslices + 31) / 32 * 32;  // equal slices, multiples of 32 columns
    if (width > cap) width = cap;
    // the slice must also leave room for the pipeline stages and the epilogue prefetch buffers: shrink until a plan fits
    int32_t any_accum = 0;
    for (int s = 0; s < n_o && o_accum; ++s) any_accum |= o_accum[s];
    while (true) {
        const int probe = width < N ? width : N;
        if (tc_launch_slice(dtype, M, K, probe, n_a, a_ptr, a_ld, a_width, a_aux, a_aux_ld, act, Wpacked, Wpacked, 1, o_ptr, o_ld, &probe, &any_accum, epi,
                            aux, aux_ld, st, nonlin, /*dry=*/true) == 0)
            break;
        if (width <= 32) return -1;
        width = (width / 2 + 31) / 32 * 32;
    }
    const uint8_t* hi = reinterpret_cast<const uint8_t*>(Wpacked);
    const uint8_t* lo = hi + (size_t)Npad_full * K * 2;
    for (int n0 = 0; n0 < N; n0 += width) {
        const int ns = (N - n0 < width) ? (N - n0) : width;
        // output sub-segments covered by [n0, n0 + ns)
        void* so_ptr[AB2_MAX_SEG];
        int64_t so_ld[AB2_MAX_SEG];
        int32_t so_w[AB2_MAX_SEG], so_acc[AB2_MAX_SEG];
        int cnt = 0, seg_lo = 0;
        for (int s = 0; s < n_o; ++s) {
            const int seg_hi = seg_lo + o_width[s];
            const int a = n0 > seg_lo ? n0 : seg_lo, b = (n0 + ns) < seg_hi ? (n0 + ns) : seg_hi;
            if (a < b) {
                so_ptr[cnt] = reinterpret_cast<uint8_t*>(o_ptr[s]) + (size_t)(a - seg_lo) * esz;
                so_ld[cnt] = o_ld[s];
                so_w[cnt] = b - a;
                so_acc[cnt] = o_accum ? o_accum[s] : 0;
                ++cnt;
            }
            seg_lo = seg_hi;
        }
        const void* aux_s = aux ? reinterpret_cast<const uint8_t*>(aux) + (size_t)n0 * esz : nullptr;
        const int rc = tc_launch_slice(dtype, M, K, ns, n_a, a_ptr, a_ld, a_width, a_aux, a_aux_ld, act, hi + (size_t)n0 * K * 2,
                                       lo + (size_t)n0 * K * 2, cnt, so_ptr, so_ld, so_w, so_acc, epi, aux_s, aux_ld, st, nonlin);
        if (rc != 0) return n0 == 0 ? -1 : 1;  // a later slice failing would leave a half-written output: report an error
    }
    return 0;
}

// Fused two-layer MLP (mlp2_kernel); contract in include/allegro_b200.h.  Returns AB2_NOT_ELIGIBLE, with nothing
// enqueued and no error set, for a case the kernel does not take: the caller then runs two ab2_linear_nl launches.
extern "C" int ab2_mlp2_nl(int dtype, int backward, int64_t M, int K, int H, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                           const int32_t* a_width, const void* W1_packed, const void* W2_packed, const void* w1_row, void* pre, int64_t pre_ld,
                           int n_o, void* const* o_ptr, const int64_t* o_ld, const int32_t* o_width, const int32_t* o_accum, void* stream,
                           int nonlin) {
    AB2_CHECK_ARG(nonlin == AB2_NL_SILU || nonlin == AB2_NL_MISH || nonlin == AB2_NL_GELU, "nonlinearity");
    AB2_CHECK_ARG(n_a >= 1 && n_a <= AB2_MAX_SEG && n_o >= 1 && n_o <= AB2_MAX_SEG, "segment count");
    AB2_CHECK_ARG(K > 0 && H > 0 && N > 0 && pre && pre_ld >= H, "shape");
    int ks = 0, ns = 0;
    for (int s = 0; s < n_a; ++s) {
        AB2_CHECK_ARG(a_ptr[s] && a_width[s] > 0 && a_ld[s] >= a_width[s], "A segment");
        ks += a_width[s];
    }
    for (int s = 0; s < n_o; ++s) {
        AB2_CHECK_ARG(o_ptr[s] && o_width[s] > 0 && o_ld[s] >= o_width[s], "output segment");
        ns += o_width[s];
    }
    AB2_CHECK_ARG(ks == K, "A segment widths must sum to K");
    AB2_CHECK_ARG(ns == N, "output segment widths must sum to N");
    const bool rank1 = w1_row != nullptr;
    AB2_CHECK_ARG(!rank1 || (backward && K == 1 && n_a == 1), "rank-1 mode is the backward of a single output column");
    if (M == 0) return 0;
    // ---- eligibility ----
    auto al16 = [](const void* ptr, int64_t ld) { return (reinterpret_cast<uintptr_t>(ptr) % 16) == 0 && (ld * 4) % 16 == 0; };
    if (dtype != AB2_F32 || !g_ab2_opt_linear_tc || !g_ab2_opt_linear_tma || !tc_encode_fn()) return AB2_NOT_ELIGIBLE;
    if (H % 32 != 0 || H > MLP2_MAX_H || !W2_packed || M >= ((int64_t)1 << 31) || !al16(pre, pre_ld)) return AB2_NOT_ELIGIBLE;
    if (rank1) {
        if (reinterpret_cast<uintptr_t>(w1_row) % 16 != 0) return AB2_NOT_ELIGIBLE;
    } else {
        if (!W1_packed || K % KC != 0 || K > MAX_K) return AB2_NOT_ELIGIBLE;
        for (int s = 0; s < n_a; ++s)
            if (a_width[s] % KC != 0 || !al16(a_ptr[s], a_ld[s])) return AB2_NOT_ELIGIBLE;
    }
    // stage-2 column chunks: equal, multiples of 32, <= MLP2_CHUNK
    const int nchunks = (N + MLP2_CHUNK - 1) / MLP2_CHUNK;
    if (nchunks > MLP2_MAX_CHUNKS) return AB2_NOT_ELIGIBLE;
    const int cwidth = ((N + nchunks - 1) / nchunks + 31) / 32 * 32;
    const int w2_npad = tc_npad(N);
    // shared-memory plan: 2 converter groups, deepest {NR raw slots, cn canonical stages} that fits
    int num_sms = 0, max_smem = 0;
    tc_device_limits(num_sms, max_smem);
    const size_t fixed = 1024 + (rank1 ? 0 : (size_t)2 * H * K * 2) + (size_t)2 * w2_npad * H * 2 + (size_t)4 * 64 * H * 2 + EPI_BYTES + MLP2_TAIL;
    const int plans[4][2] = {{4, 4}, {2, 4}, {4, 2}, {2, 2}};  // {NR, cn}
    // (rank-1: no ring at all, NR = nstage = 0 -- the kernel lays out W1, W2, ... behind NR raw slots and nstage stages)
    int NR = 0, nstage = 0;
    size_t smem = rank1 ? fixed : 0;
    for (int q = 0; q < 4 && !rank1 && !NR; ++q) {
        const size_t need = fixed + (size_t)(plans[q][0] * TMA_BOX_BYTES + plans[q][1] * 2 * STAGE_HALF);
        if (need <= (size_t)max_smem) { NR = plans[q][0]; nstage = plans[q][1]; smem = need; }
    }
    if (smem == 0 || smem > (size_t)max_smem) return AB2_NOT_ELIGIBLE;

    Mlp2Params q;
    memset(&q, 0, sizeof(q));
    TmaMaps maps;
    memset(&maps, 0, sizeof(maps));
    const int64_t num_tiles = (M + BM - 1) / BM;
    TcParams& p = q.s1;
    p.M = M; p.K = K; p.N = H; p.Npad = H; p.n_a = n_a; p.act = AB2_ACT_NONE; p.epi = AB2_EPI_NONE;
    p.num_tiles = num_tiles; p.nstage = nstage;
    for (int s = 0; s < n_a; ++s) { p.a[s].ptr = a_ptr[s]; p.a[s].ld = a_ld[s]; p.a[s].width = a_width[s]; }
    if (rank1) {
        q.gout1 = reinterpret_cast<const float*>(a_ptr[0]);
        q.gout1_ld = a_ld[0];
        q.w1row = reinterpret_cast<const float*>(w1_row);
    } else {
        p.Wpacked = W1_packed;
        p.Wlo = reinterpret_cast<const uint8_t*>(W1_packed) + (size_t)H * K * 2;
        for (int s = 0; s < n_a; ++s)
            if (!tc_make_map(&maps.a[s], a_ptr[s], a_ld[s], a_width[s], M)) return AB2_NOT_ELIGIBLE;
    }
    if (backward) {
        q.backward = 1;
        q.pre = reinterpret_cast<const float*>(pre);
        q.pre_ld = pre_ld;
    } else {
        p.n_o = 1;
        p.o[0].ptr = pre; p.o[0].ld = pre_ld; p.o[0].width = H;
    }
    q.w2_npad = w2_npad;
    q.n2 = 0;
    for (int n0 = 0; n0 < N; n0 += cwidth, ++q.n2) {
        const int nc = (N - n0 < cwidth) ? (N - n0) : cwidth;
        TcParams& p2 = q.s2[q.n2];
        p2.M = M; p2.K = H; p2.N = nc; p2.Npad = tc_npad(nc); p2.epi = AB2_EPI_NONE; p2.num_tiles = num_tiles;
        q.n0[q.n2] = n0;
        // output segments covered by [n0, n0 + nc)
        int seg_lo = 0;
        for (int s = 0; s < n_o; ++s) {
            const int seg_hi = seg_lo + o_width[s];
            const int a = n0 > seg_lo ? n0 : seg_lo, b = (n0 + nc) < seg_hi ? (n0 + nc) : seg_hi;
            if (a < b) {
                TcSeg& o = p2.o[p2.n_o++];
                o.ptr = reinterpret_cast<float*>(o_ptr[s]) + (a - seg_lo);
                o.ld = o_ld[s];
                o.width = b - a;
                o.accum = o_accum ? o_accum[s] : 0;
            }
            seg_lo = seg_hi;
        }
    }
    q.s2[0].Wpacked = W2_packed;  // the whole W2 image (hi, then lo) is staged once
    q.s2[0].Wlo = reinterpret_cast<const uint8_t*>(W2_packed) + (size_t)w2_npad * H * 2;

    const unsigned grid = (unsigned)((num_tiles < num_sms) ? num_tiles : num_sms);
    cudaStream_t st = (cudaStream_t)stream;
    auto go = [&](auto kern) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return AB2_NOT_ELIGIBLE;
        }
        kern<<<grid, NTHREADS, smem, st>>>(q, maps, NR);
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    };
    return tc_with_nl(nonlin, [&](auto nl) -> int {
        constexpr int NL = decltype(nl)::value;
        switch (H / 32) {
            case 1: return go(mlp2_kernel<1, NL>);
            case 2: return go(mlp2_kernel<2, NL>);
        }
        return AB2_NOT_ELIGIBLE;
    });
}

extern "C" int ab2_mlp2(int dtype, int backward, int64_t M, int K, int H, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                        const int32_t* a_width, const void* W1_packed, const void* W2_packed, const void* w1_row, void* pre, int64_t pre_ld, int n_o,
                        void* const* o_ptr, const int64_t* o_ld, const int32_t* o_width, const int32_t* o_accum, void* stream) {
    return ab2_mlp2_nl(dtype, backward, M, K, H, N, n_a, a_ptr, a_ld, a_width, W1_packed, W2_packed, w1_row, pre, pre_ld, n_o, o_ptr, o_ld, o_width,
                       o_accum, stream, AB2_NL_SILU);
}

// Gradient GEMM of the scalar-embed MLP + radial adjoint (radial_adjoint_tma_kernel); contract in include/allegro_b200.h.
// Returns AB2_NOT_ELIGIBLE, with nothing enqueued and no error set, for a case the kernel does not take: the caller then
// runs ab2_linear and ab2_radial_pq_bwd_nl.
extern "C" int ab2_radial_pq_bwd_gemm(int dtype, int64_t M, int K, int H, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                                      const int32_t* a_width, const void* W_packed, int num_bessels, double p_cut, const void* vec,
                                      const int32_t* ctr, const int32_t* nbr, const int32_t* types, const void* rmax_table, int num_types,
                                      const void* bessel_w, const void* PQ, void* gvec, void* stream, int nonlin) {
    AB2_CHECK_ARG(nonlin == AB2_NL_SILU || nonlin == AB2_NL_MISH || nonlin == AB2_NL_GELU, "nonlinearity");
    AB2_CHECK_ARG(M >= 0, "shape");
    if (M == 0) return 0;  // (empty operands may come with null pointers)
    AB2_CHECK_ARG(n_a >= 1 && n_a <= AB2_MAX_SEG, "segment count");
    AB2_CHECK_ARG(K > 0 && H > 0 && num_types > 0, "shape");
    int ks = 0;
    for (int s = 0; s < n_a; ++s) {
        AB2_CHECK_ARG(a_ptr[s] && a_width[s] > 0 && a_ld[s] >= a_width[s], "A segment");
        ks += a_width[s];
    }
    AB2_CHECK_ARG(ks == K, "A segment widths must sum to K");
    AB2_CHECK_ARG(vec && ctr && nbr && types && rmax_table && bessel_w && PQ && gvec, "null pointer");
    // ---- eligibility ----
    auto al16 = [](const void* ptr, int64_t ld) { return (reinterpret_cast<uintptr_t>(ptr) % 16) == 0 && (ld * 4) % 16 == 0; };
    if (dtype != AB2_F32 || !g_ab2_opt_linear_tc || !g_ab2_opt_linear_tma || !tc_encode_fn()) return AB2_NOT_ELIGIBLE;
    if (num_bessels != RADJ_NB || (H != 32 && H != 64) || !W_packed || K % KC != 0 || K > MAX_K || M >= ((int64_t)1 << 31))
        return AB2_NOT_ELIGIBLE;
    if ((size_t)num_types * num_types * RADJ_NB * H * 4 > (size_t)EPI_BYTES) return AB2_NOT_ELIGIBLE;  // PQ in the staging area
    for (int s = 0; s < n_a; ++s)
        if (a_width[s] % KC != 0 || !al16(a_ptr[s], a_ld[s])) return AB2_NOT_ELIGIBLE;
    // shared-memory plan of linear_tma_kernel with four converter groups: deepest {NR raw slots, cn canonical stages}
    int num_sms = 0, max_smem = 0;
    tc_device_limits(num_sms, max_smem);
    const int w_bytes = 2 * H * K * 2;
    const int plans[2][2] = {{8, 4}, {4, 4}};  // {NR, cn}
    int NR = 0, nstage = 0;
    size_t smem = 0;
    for (int q = 0; q < 2 && !NR; ++q) {
        const size_t need = 1024 + ((w_bytes + 127) & ~127) + (size_t)plans[q][1] * 2 * STAGE_HALF + EPI_BYTES + TAIL_BYTES +
                            (size_t)plans[q][0] * TMA_BOX_BYTES;
        if (need <= (size_t)max_smem) { NR = plans[q][0]; nstage = plans[q][1]; smem = need; }
    }
    if (!NR) return AB2_NOT_ELIGIBLE;

    TcParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.K = K; p.N = H; p.Npad = H; p.n_a = n_a; p.act = AB2_ACT_NONE; p.epi = AB2_EPI_NONE;
    p.Wpacked = W_packed; p.Wlo = reinterpret_cast<const uint8_t*>(W_packed) + (size_t)H * K * 2;
    p.num_tiles = (M + BM - 1) / BM; p.nstage = nstage; p.debug = g_ab2_opt_tc_debug;
    TmaMaps maps;
    memset(&maps, 0, sizeof(maps));
    for (int s = 0; s < n_a; ++s) {
        p.a[s].ptr = a_ptr[s]; p.a[s].ld = a_ld[s]; p.a[s].width = a_width[s];
        if (!tc_make_map(&maps.a[s], a_ptr[s], a_ld[s], a_width[s], M)) return AB2_NOT_ELIGIBLE;
    }
    RadialAdjParams ra;
    ra.vec = reinterpret_cast<const float*>(vec); ra.ctr = ctr; ra.nbr = nbr; ra.types = types;
    ra.rmax_table = reinterpret_cast<const float*>(rmax_table); ra.bw = reinterpret_cast<const float*>(bessel_w);
    ra.PQ = reinterpret_cast<const float*>(PQ); ra.gvec = reinterpret_cast<float*>(gvec);
    ra.num_types = num_types; ra.p = (float)p_cut;

    const unsigned grid = (unsigned)((p.num_tiles < num_sms) ? p.num_tiles : num_sms);
    cudaStream_t st = (cudaStream_t)stream;
    auto go = [&](auto kern) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return AB2_NOT_ELIGIBLE;
        }
        kern<<<grid, NTHREADS, smem, st>>>(p, maps, NR, ra);
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    };
    return tc_with_nl(nonlin, [&](auto nl) -> int {
        constexpr int NL = decltype(nl)::value;
        return H == 32 ? go(radial_adjoint_tma_kernel<4, 1, NL>) : go(radial_adjoint_tma_kernel<4, 2, NL>);
    });
}

// Radial embedding + the scalar-embed MLP's folded last layer (radial_embed_fwd_kernel); contract in include/allegro_b200.h.
// Returns AB2_NOT_ELIGIBLE, with nothing enqueued and no error set, for a case the kernel does not take: the caller then
// runs ab2_radial_pq_fwd and ab2_linear_nl.
extern "C" int ab2_radial_embed_fwd(int dtype, int64_t M, int H, int N, const void* W_packed, int num_bessels, double p_cut, const void* vec,
                                    const int32_t* ctr, const int32_t* nbr, const int32_t* types, const void* rmax_table, int num_types,
                                    const void* bessel_w, const void* PQ, int n_o, void* const* o_ptr, const int64_t* o_ld, const int32_t* o_width,
                                    void* stream, int nonlin) {
    AB2_CHECK_ARG(nonlin == AB2_NL_SILU || nonlin == AB2_NL_MISH || nonlin == AB2_NL_GELU, "nonlinearity");
    AB2_CHECK_ARG(M >= 0, "shape");
    if (M == 0) return 0;  // (empty operands may come with null pointers)
    AB2_CHECK_ARG(n_o >= 1 && n_o <= AB2_MAX_SEG, "segment count");
    AB2_CHECK_ARG(H > 0 && N > 0 && num_types > 0, "shape");
    int ns = 0;
    for (int s = 0; s < n_o; ++s) {
        AB2_CHECK_ARG(o_ptr[s] && o_width[s] > 0 && o_ld[s] >= o_width[s], "output segment");
        ns += o_width[s];
    }
    AB2_CHECK_ARG(ns == N, "output segment widths must sum to N");
    AB2_CHECK_ARG(W_packed && vec && ctr && nbr && types && rmax_table && bessel_w && PQ, "null pointer");
    // ---- eligibility ----
    if (dtype != AB2_F32 || !g_ab2_opt_linear_tc || !g_ab2_opt_linear_tma) return AB2_NOT_ELIGIBLE;
    if (num_bessels != RADJ_NB || (H != 32 && H != 64) || N > REMB_MAX_CHUNKS * MAX_N || M >= ((int64_t)1 << 31)) return AB2_NOT_ELIGIBLE;
    for (int s = 0; s < n_o; ++s)  // every 32-column chunk inside one segment, on the coalesced epilogue path
        if (o_width[s] % 32 != 0 || (reinterpret_cast<uintptr_t>(o_ptr[s]) % 16) != 0 || (o_ld[s] * 4) % 16 != 0) return AB2_NOT_ELIGIBLE;
    const int Npad = tc_npad(N);
    const int w_half = Npad * H * 2;
    const size_t pq_bytes = (size_t)num_types * num_types * (RADJ_NB * H + 4) * 4;
    const size_t smem = (size_t)2 * w_half + (size_t)4 * BM * H * 2 + EPI_BYTES + ((pq_bytes + 15) & ~(size_t)15) + 4 * 8 +
                        REMB_MAX_CHUNKS * MAX_CHUNK * sizeof(ChunkInfo);
    int num_sms = 0, max_smem = 0;
    tc_device_limits(num_sms, max_smem);
    if (smem > (size_t)max_smem) return AB2_NOT_ELIGIBLE;  // PQ beyond what is left next to W_fold and the A tiles

    RadialEmbedParams q;
    memset(&q, 0, sizeof(q));
    q.M = M; q.num_tiles = (M + BM - 1) / BM;
    // column chunks: the slices of ab2_linear_tc_try (equal, multiples of 32, <= MAX_N), so each chunk runs the wgmma shape
    // of the launch it replaces
    const int nchunks = (N + MAX_N - 1) / MAX_N;
    const int cwidth = ((N + nchunks - 1) / nchunks + 31) / 32 * 32;
    for (int n0 = 0; n0 < N; n0 += cwidth, ++q.n_chunks) {
        const int nc = (N - n0 < cwidth) ? (N - n0) : cwidth;
        TcParams& pc = q.s[q.n_chunks];
        pc.M = M; pc.K = H; pc.N = nc; pc.Npad = tc_npad(nc); pc.epi = AB2_EPI_NONE; pc.num_tiles = q.num_tiles;
        q.n0[q.n_chunks] = n0;
        int seg_lo = 0;
        for (int s = 0; s < n_o; ++s) {  // output segments covered by [n0, n0 + nc)
            const int seg_hi = seg_lo + o_width[s];
            const int a = n0 > seg_lo ? n0 : seg_lo, b = (n0 + nc) < seg_hi ? (n0 + nc) : seg_hi;
            if (a < b) {
                TcSeg& o = pc.o[pc.n_o++];
                o.ptr = reinterpret_cast<float*>(o_ptr[s]) + (a - seg_lo);
                o.ld = o_ld[s];
                o.width = b - a;
            }
            seg_lo = seg_hi;
        }
    }
    q.w_half = w_half;
    q.W = W_packed;
    q.vec = reinterpret_cast<const float*>(vec); q.ctr = ctr; q.nbr = nbr; q.types = types;
    q.rmax_table = reinterpret_cast<const float*>(rmax_table); q.bw = reinterpret_cast<const float*>(bessel_w);
    q.PQ = reinterpret_cast<const float*>(PQ); q.num_types = num_types; q.p = (float)p_cut;

    const unsigned grid = (unsigned)((q.num_tiles < num_sms) ? q.num_tiles : num_sms);
    cudaStream_t st = (cudaStream_t)stream;
    auto go = [&](auto kern) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return AB2_NOT_ELIGIBLE;
        }
        kern<<<grid, NTHREADS, smem, st>>>(q);
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    };
    return tc_with_nl(nonlin, [&](auto nl) -> int {
        constexpr int NL = decltype(nl)::value;
        return H == 32 ? go(radial_embed_fwd_kernel<1, NL>) : go(radial_embed_fwd_kernel<2, NL>);
    });
}

// Last latent MLP + readout MLP (mlp2_readout_fwd_kernel / mlp2_readout_bwd_kernel); contract in include/allegro_b200.h.
// Returns AB2_NOT_ELIGIBLE, with nothing enqueued and no error set, for a case the kernels do not take: the caller then
// runs the two MLPs as two ab2_mlp2_nl (or ab2_linear_nl) calls.
extern "C" int ab2_mlp2_readout_nl(int dtype, int backward, int64_t M, int P, int S, int U, int H, void* x, int64_t x_ld, void* s, int64_t s_ld,
                                   void* xl, int64_t xl_ld, void* pre_l, int64_t pre_l_ld, void* pre_r, int64_t pre_r_ld, void* ez, int64_t ez_ld,
                                   const void* const* w_packed, const void* w2_ro, void* stream, int nonlin) {
    AB2_CHECK_ARG(nonlin == AB2_NL_SILU || nonlin == AB2_NL_MISH || nonlin == AB2_NL_GELU, "nonlinearity");
    AB2_CHECK_ARG(P > 0 && S > 0 && U > 0 && H > 0 && M >= 0, "shape");
    AB2_CHECK_ARG(x && s && pre_l && pre_r && ez && w2_ro && w_packed && (backward || xl), "null pointer");
    AB2_CHECK_ARG(x_ld >= P && s_ld >= U && (backward || xl_ld >= S) && pre_l_ld >= H && pre_r_ld >= H && ez_ld >= 1, "leading dimension");
    if (M == 0) return 0;
    // ---- eligibility ----
    const int n_w = backward ? 3 : 4;
    auto al16 = [](const void* ptr, int64_t ld) { return (reinterpret_cast<uintptr_t>(ptr) % 16) == 0 && (ld * 4) % 16 == 0; };
    if (dtype != AB2_F32 || !g_ab2_opt_linear_tc || !g_ab2_opt_linear_tma || (!backward && !tc_encode_fn())) return AB2_NOT_ELIGIBLE;
    if (H != RO_H || S != RO_H || P % KC != 0 || U % KC != 0 || P + U > MAX_K || M >= ((int64_t)1 << 31)) return AB2_NOT_ELIGIBLE;
    if (!al16(x, x_ld) || !al16(s, s_ld) || (!backward && !al16(xl, xl_ld)) || !al16(pre_l, pre_l_ld) || !al16(pre_r, pre_r_ld) ||
        reinterpret_cast<uintptr_t>(w2_ro) % 16 != 0)
        return AB2_NOT_ELIGIBLE;
    for (int i = 0; i < n_w; ++i)
        if (!w_packed[i]) return AB2_NOT_ELIGIBLE;

    Mlp2RoParams q;
    memset(&q, 0, sizeof(q));
    const int64_t num_tiles = (M + BM - 1) / BM;
    q.P = P;
    q.w2ro = reinterpret_cast<const float*>(w2_ro);
    q.ez = reinterpret_cast<float*>(ez);
    q.ez_ld = ez_ld;
    for (int i = 0; i < n_w; ++i) q.w[i] = w_packed[i];
    TcParams& p = q.s1;
    p.M = M; p.num_tiles = num_tiles;
    auto out1 = [&](TcParams& o, void* ptr, int64_t ld, int n) {  // one output segment of n columns, plain stores
        o.M = M; o.K = H; o.N = n; o.Npad = n; o.epi = AB2_EPI_NONE; o.num_tiles = num_tiles;
        o.n_o = 1; o.o[0].ptr = ptr; o.o[0].ld = ld; o.o[0].width = n;
    };
    int num_sms = 0, max_smem = 0;
    tc_device_limits(num_sms, max_smem);
    const unsigned grid = (unsigned)((num_tiles < num_sms) ? num_tiles : num_sms);
    cudaStream_t st = (cudaStream_t)stream;
    auto go = [&](auto kern, size_t smem, auto... args) -> int {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();
            return AB2_NOT_ELIGIBLE;
        }
        kern<<<grid, NTHREADS, smem, st>>>(q, args...);
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    };

    if (backward) {
        // output chunks of [gX[:, :P] | gs]: the prefix, then gs, each in pieces of at most 64 columns
        for (int seg = 0; seg < 2; ++seg) {
            const int lo = seg ? P : 0, hi = seg ? P + U : P;
            for (int n0 = lo; n0 < hi; n0 += 64) {
                if (q.n_chunks == RO_MAX_CHUNKS) return AB2_NOT_ELIGIBLE;
                const int nc = hi - n0 < 64 ? hi - n0 : 64;
                float* base = seg ? reinterpret_cast<float*>(s) + (n0 - P) : reinterpret_cast<float*>(x) + n0;
                out1(q.o[q.n_chunks], base, seg ? s_ld : x_ld, nc);
                q.n0[q.n_chunks++] = n0;
            }
        }
        q.w_half[0] = (P + S) * H * 2;  // W1_ro^T: K = H, N = P + S
        q.w_half[1] = H * S * 2;        // W2_lat^T: K = S, N = H
        q.w_half[2] = (P + U) * H * 2;  // W1_lat^T: K = H, N = P + U
        q.pre_l = reinterpret_cast<const float*>(pre_l); q.pre_l_ld = pre_l_ld;
        q.pre_r = reinterpret_cast<const float*>(pre_r); q.pre_r_ld = pre_r_ld;
        const size_t smem = (size_t)2 * (q.w_half[0] + q.w_half[1] + q.w_half[2]) + (size_t)12 * RO_TILE + EPI_BYTES + RO_TAIL;
        if (smem > (size_t)max_smem) return AB2_NOT_ELIGIBLE;
        return tc_with_nl(nonlin, [&](auto nl) { return go(mlp2_readout_bwd_kernel<decltype(nl)::value>, smem); });
    }

    p.K = P + U; p.N = H; p.Npad = H; p.n_a = 2; p.act = AB2_ACT_NONE; p.epi = AB2_EPI_NONE;
    p.a[0].ptr = x; p.a[0].ld = x_ld; p.a[0].width = P;
    p.a[1].ptr = s; p.a[1].ld = s_ld; p.a[1].width = U;
    p.Wpacked = w_packed[0];
    p.n_o = 1; p.o[0].ptr = pre_l; p.o[0].ld = pre_l_ld; p.o[0].width = H;
    out1(q.o[0], xl, xl_ld, S);
    out1(q.o[1], pre_r, pre_r_ld, H);
    q.w_half[0] = H * (P + U) * 2;  // W1_lat: K = P + U, N = H
    q.w_half[1] = S * H * 2;        // W2_lat: K = H, N = S
    q.w_half[2] = H * P * 2;        // W1_ro[:P]: K = P, N = H
    q.w_half[3] = H * S * 2;        // W1_ro[P:]: K = S, N = H
    p.Wlo = reinterpret_cast<const uint8_t*>(w_packed[0]) + q.w_half[0];
    // shared-memory plan: 2 converter groups, deepest {NR raw slots, cn canonical stages} that fits
    const size_t fixed = 1024 + (size_t)2 * (q.w_half[0] + q.w_half[1] + q.w_half[2] + q.w_half[3]) + (size_t)4 * RO_TILE + EPI_BYTES + RO_TAIL;
    const int plans[4][2] = {{4, 4}, {2, 4}, {4, 2}, {2, 2}};  // {NR, cn}
    int NR = 0;
    size_t smem = 0;
    for (int i = 0; i < 4 && !NR; ++i) {
        const size_t need = fixed + (size_t)(plans[i][0] * TMA_BOX_BYTES + plans[i][1] * 2 * STAGE_HALF);
        if (need <= (size_t)max_smem) { NR = plans[i][0]; p.nstage = plans[i][1]; smem = need; }
    }
    if (!NR) return AB2_NOT_ELIGIBLE;
    TmaMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (!tc_make_map(&maps.a[0], x, x_ld, P, M) || !tc_make_map(&maps.a[1], s, s_ld, U, M)) return AB2_NOT_ELIGIBLE;
    return tc_with_nl(nonlin, [&](auto nl) { return go(mlp2_readout_fwd_kernel<decltype(nl)::value>, smem, maps, NR); });
}

extern "C" int ab2_mlp2_readout(int dtype, int backward, int64_t M, int P, int S, int U, int H, void* x, int64_t x_ld, void* s, int64_t s_ld,
                                void* xl, int64_t xl_ld, void* pre_l, int64_t pre_l_ld, void* pre_r, int64_t pre_r_ld, void* ez, int64_t ez_ld,
                                const void* const* w_packed, const void* w2_ro, void* stream) {
    return ab2_mlp2_readout_nl(dtype, backward, M, P, S, U, H, x, x_ld, s, s_ld, xl, xl_ld, pre_l, pre_l_ld, pre_r, pre_r_ld, ez, ez_ld, w_packed, w2_ro,
                               stream, AB2_NL_SILU);
}

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

#include "common.cuh"

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
template <typename TSrc, bool SPLIT, int NCH>
__device__ __forceinline__ void tc_consumer_role(const TcParams& p, const TcCtx& c, int cw, int lane) {
    const int wg = cw >> 2, w4 = cw & 3;
    const int nkb = c.nkb, stage_bytes = c.stage_bytes, w_half = c.w_half;
    const uint32_t sW_u = smem_u32(c.sW);
    const uint32_t w_sbo = (uint32_t)(p.K / 8) * 128;  // bytes between 8-column (n) groups of W
    constexpr uint32_t A_SBO = (KC / 8) * 128;         // bytes between 8-row groups of a stage
    float* stg = c.sEpi + cw * 16 * EPI_LD;
    int stage = 0;
    uint32_t phase = 0;
    float acc[16 * NCH];
    for (int64_t tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
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
                if constexpr (SPLIT) {
                    const uint64_t da_lo = make_desc(a_hi + STAGE_HALF + ks * 256, 128, A_SBO);
                    const uint64_t db_lo = make_desc(wk + w_half, 128, w_sbo);
                    wgmma_bf16<NCH>(acc, da_lo, db_hi, 1u);
                    wgmma_bf16<NCH>(acc, da_hi, db_lo, 1u);
                }
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

        // ---- epilogue: this warp's 16 rows, one 32-column chunk at a time ----
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
            if (p.epi == AB2_EPI_MUL_DSILU) {
                const TSrc* ax = (const TSrc*)p.aux + m * p.aux_ld + c0;
                if (sizeof(TSrc) == 4 && c0 + 16 <= p.N && ((reinterpret_cast<uintptr_t>(ax) & 15) == 0)) {
                    const float4* a4 = reinterpret_cast<const float4*>(ax);
#pragma unroll
                    for (int t = 0; t < 4; ++t) {
                        const float4 x = __ldg(a4 + t);
                        v[4 * t] *= dsilu_f(x.x); v[4 * t + 1] *= dsilu_f(x.y); v[4 * t + 2] *= dsilu_f(x.z); v[4 * t + 3] *= dsilu_f(x.w);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < 16; ++j)
                        if (c0 + j < p.N) v[j] *= dsilu_f(to_acc<float>(ax[j]));
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
            const ChunkInfo ci = c.sChunk[ch];
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
                if (p.epi == AB2_EPI_MUL_DSILU) {
                    float4 ax[4];
                    const float* ab = ci.aptr + m_base * p.aux_ld + c4 * 4;
                    const uint32_t al = (uint32_t)p.aux_ld;
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) ax[itr] = ldg128_nc(ab + (uint32_t)row_of(itr) * al);
#pragma unroll
                    for (int itr = 0; itr < 4; ++itr) {
                        x[itr].x *= dsilu_fast(ax[itr].x); x[itr].y *= dsilu_fast(ax[itr].y);
                        x[itr].z *= dsilu_fast(ax[itr].z); x[itr].w *= dsilu_fast(ax[itr].w);
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
            } else {
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

template <typename TSrc, bool SPLIT, int NCH>
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
                        for (int t = 0; t < 8; ++t) v[i][t] *= dsilu_fast(w[t]);
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
                    for (int t = 0; t < 8; ++t) v[i][t] = silu_fast(v[i][t]);
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
        tc_consumer_role<TSrc, SPLIT, NCH>(p, ctx, warp - NPROD, lane);
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

// G converter groups of 8/G warps.  A raw slot and a canonical stage must always be consumed / produced by the SAME group
// (NR % G == 0 and nstage % G == 0, checked on the host): a group then never waits more than one mbarrier phase ahead
// of its own slot.  (With slots shared between groups a group's first wait can be for the SECOND fill of a slot whose
// first fill has not completed yet -- the parity wait returns immediately and the pipeline falls apart.)
template <int G, int NCH>
__global__ void __launch_bounds__(NTHREADS, 1) linear_tma_kernel(const TcParams p, const __grid_constant__ TmaMaps maps, int NR) {
    constexpr int WPG = NPROD / G;      // warps per converter group
    constexpr int RGW = 16 / WPG;       // 8-row groups of a stage handled by one warp
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
    auto rfull_bar = [&](int s) { return rbar0 + 8u * s; };
    const int nkb = p.K / KC;

    // ---- one-time setup ----
    if (threadIdx.x == 0) {
        for (int s = 0; s < NSTAGE; ++s) {
            mbar_init(bar0 + 8u * s, WPG * 32);          // canonical stage full: the warps of one converter group
            mbar_init(bar0 + 8u * (NSTAGE + s), NCONS);  // empty: one arrive per consumer warp
        }
        for (int s = 0; s < 8; ++s) mbar_init(rfull_bar(s), 1);  // expect_tx arrive of the issuing lane
        fence_barrier_init();
    }
    if (threadIdx.x < MAX_K / 32) {
        int kk = threadIdx.x * KC;
        int4 ent = make_int4(-1, 0, 0, 0);
#pragma unroll
        for (int sgi = 0; sgi < AB2_MAX_SEG; ++sgi) {
            if (sgi < p.n_a && ent.x < 0 && kk < p.K) {
                if (kk < p.a[sgi].width) ent = make_int4(sgi, kk, p.a[sgi].aux ? 1 : 0, 0);
                kk -= p.a[sgi].width;
            }
        }
        sKseg[threadIdx.x] = ent;
    } else if (threadIdx.x >= 64 && threadIdx.x < 64 + MAX_CHUNK) {
        sChunk[threadIdx.x - 64] = tc_chunk_info<TSrc>(p, (threadIdx.x - 64) * 32);
    }
    {
        const uint4* src = reinterpret_cast<const uint4*>(p.Wpacked);
        uint4* dst = reinterpret_cast<uint4*>(sW);
        for (int e = threadIdx.x; e < w_half / 16; e += NTHREADS) dst[e] = __ldg(src + e);
        const uint4* srcl = reinterpret_cast<const uint4*>(p.Wlo);
        uint4* dstl = reinterpret_cast<uint4*>(sW + w_half);
        for (int e = threadIdx.x; e < w_half / 16; e += NTHREADS) dstl[e] = __ldg(srcl + e);
    }
    fence_proxy_async();
    __syncthreads();
    TcCtx ctx;
    ctx.sW = sW; ctx.sA = sA; ctx.sEpi = sEpi; ctx.sChunk = sChunk; ctx.bar0 = bar0;
    ctx.nkb = nkb; ctx.stage_bytes = stage_bytes; ctx.w_half = w_half;
    const int64_t my_tiles = (p.num_tiles > blockIdx.x) ? (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const int64_t total = my_tiles * nkb;

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

    if (warp >= NPROD) {
        tc_consumer_role<TSrc, SPLIT, NCH>(p, ctx, warp - NPROD, lane);
    } else {
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
                    v[i][0] *= dsilu_fast(x.x); v[i][1] *= dsilu_fast(x.y); v[i][2] *= dsilu_fast(x.z); v[i][3] *= dsilu_fast(x.w);
                    v[i][4] *= dsilu_fast(y.x); v[i][5] *= dsilu_fast(y.y); v[i][6] *= dsilu_fast(y.z); v[i][7] *= dsilu_fast(y.w);
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
                    for (int t = 0; t < 8; ++t) v[i][t] = silu_fast(v[i][t]);
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

static int tc_launch_tma(TcParams& p, int w_bytes, int stage_bytes, int max_smem, unsigned grid, cudaStream_t st, bool dry) {
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
    switch ((G == 4 ? 4 : 0) + p.Npad / 32) {
        case 1: return go(linear_tma_kernel<2, 1>);
        case 2: return go(linear_tma_kernel<2, 2>);
        case 3: return go(linear_tma_kernel<2, 3>);
        case 4: return go(linear_tma_kernel<2, 4>);
        case 5: return go(linear_tma_kernel<4, 1>);
        case 6: return go(linear_tma_kernel<4, 2>);
        case 7: return go(linear_tma_kernel<4, 3>);
        case 8: return go(linear_tma_kernel<4, 4>);
    }
    return -1;
}

// One column slice [n0, n0 + N) of the GEMM with its W images resident in shared memory.
static int tc_launch_slice(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                           const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* Whi, const void* Wlo,
                           int n_o, void* const* o_ptr, const int64_t* o_ld, const int32_t* o_width, const int32_t* o_accum, int epi,
                           const void* aux, int64_t aux_ld, cudaStream_t st, bool dry = false) {
    const int has_aux = (act == AB2_ACT_MUL_DSILU && a_aux) ? 1 : 0;
    if (tc_npad(N) > MAX_N) return -1;
    static int num_sms = 0;
    static int max_smem = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    }
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
        const int rc = tc_launch_tma(p, w_bytes, stage_bytes, max_smem, grid, st, dry);
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
    switch ((split ? 4 : 0) + p.Npad / 32) {
        case 1: return go(linear_tc_kernel<bf16, false, 1>);
        case 2: return go(linear_tc_kernel<bf16, false, 2>);
        case 3: return go(linear_tc_kernel<bf16, false, 3>);
        case 4: return go(linear_tc_kernel<bf16, false, 4>);
        case 5: return go(linear_tc_kernel<float, true, 1>);
        case 6: return go(linear_tc_kernel<float, true, 2>);
        case 7: return go(linear_tc_kernel<float, true, 3>);
        case 8: return go(linear_tc_kernel<float, true, 4>);
    }
    return -1;
}

// returns 0 if launched, -1 if this call is not eligible (caller falls back to linear.cu).
// Outputs wider than MAX_N columns, or whose W image exceeds the shared-memory budget, run as column slices (one launch
// per slice, each with its W slice resident; the A rows are re-read per slice).
int ab2_linear_tc_try(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                      const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* Wpacked, int n_o, void* const* o_ptr, const int64_t* o_ld,
                      const int32_t* o_width, const int32_t* o_accum, int epi, const void* aux, int64_t aux_ld, cudaStream_t st) {
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
                            aux, aux_ld, st, /*dry=*/true) == 0)
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
                                       lo + (size_t)n0 * K * 2, cnt, so_ptr, so_ld, so_w, so_acc, epi, aux_s, aux_ld, st);
        if (rc != 0) return n0 == 0 ? -1 : 1;  // a later slice failing would leave a half-written output: report an error
    }
    return 0;
}

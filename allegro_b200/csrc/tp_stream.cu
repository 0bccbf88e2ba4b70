// Streaming tensor-product kernels: the CSR rows are staged through shared memory by the TMA unit.
//
// Reference semantics: Contracter._contract (allegro/nn/_strided/_contract.py:213-251) after the
// scatter/gather of :199-205, forward and both backward products (the Triton back-end's fwd / bwd1 /
// bwd2 tables, _flashallegro.py:347-360), on centre-sorted CSR edges and the component-major layout.
//
// Why this shape.  With centre-sorted edges everything a centre needs is CONTIGUOUS in HBM: the rows
// gVout[z0:z1][d_out][U], Vin[z0:z1][d_in][U] (or, layer 0, w0[z0:z1][n_ir][U] and Y[z0:z1][d]) and
// gamma[c][d][U].  So the "neighbour-list gather" is a handful of 1-D bulk copies
// (cp.async.bulk.shared.global, SASS UBLKCP) per stage of TE edges, issued by ONE elected producer
// thread and completed on an mbarrier -- the memory-level parallelism (NS stages x several CTAs per
// SM, 100+ KB in flight per SM) no longer depends on registers or on the number of resident warps,
// which is what limits kernels that keep M in registers or shared memory and load with plain per-thread loads.
//
// Work split.  Persistent-style grid: CTA b owns a contiguous range of centres holding ~E/grid edges
// (binary search over row_ptr), i.e. one contiguous edge stream.  Per CTA:
//   warp 2*NCH      producer : lane 0 issues the bulk copies (edge stages + gamma[c] one centre ahead),
//                              all lanes copy the small Y rows (36 B/edge, not 16-byte aligned) with
//                              4-byte cp.async completing on the same mbarrier (noinc arrive);
//   warps 0..2*NCH-1 consumers: per 32-channel chunk TWO warps (lane = channel) that split the coupling
//                              matrix M_c[i][k] = sum_nnz cgw * gamma[c][j]  by ROWS i (backward) or COLUMNS k
//                              (forward), so M and the gradient accumulator gM stay in registers
//                              (<= 45 + 45 values) at ~130 registers -> 4-5 CTAs per SM.
// The backward is ONE launch: gVin / gw0 / gY per edge and gM accumulated over the centre's row, then
// ggamma[c][j] = sum_nnz cgw * gM[i][k] once per centre -- written exactly once, no atomics, fixed order
// (deterministic), gVout / w0 / Y read exactly once.
#include <type_traits>

#include "common.cuh"
#include "tp_fast.cuh"
#include "tp_tables_generated.cuh"
#include "stream_common.cuh"

#if !defined(AB2_TP_STREAM_GROUP) || AB2_TP_STREAM_GROUP == 0  // defined once, in group 0 (see the end of this file)
int g_ab2_opt_tp_stream = 1;    // 1: use these kernels where instantiated, 0: round-1 kernels
int g_ab2_opt_tp_stream_te = 0;  // edges per stage (0 = default 8), 8 or 16
int g_ab2_opt_tp_stream_cps = 0; // cap on CTAs per SM (0 = occupancy limit)
int g_ab2_opt_tp_stream_last = 1;    // 9 -> 1 (last layer) backward through the streaming kernel instead of tp_smem + split
int g_ab2_opt_tp_stream_gytile = 1;  // layer-0 backward: gY reduced through a shared-memory tile instead of per-edge shuffles
#else
extern int g_ab2_opt_tp_stream, g_ab2_opt_tp_stream_te, g_ab2_opt_tp_stream_cps, g_ab2_opt_tp_stream_last, g_ab2_opt_tp_stream_gytile;
#endif

namespace {

// baked 9 x 9 x 9 structure packed i | j << 8 | k << 16 in constant memory: the stand-down test of a launch that follows the
// three-warp kernel (skip_if_baked) runs before any set-up and costs a few microseconds instead of the whole prologue
struct PackedTab9 {
    uint32_t v[Tab9x9x9::NNZ];
};
constexpr PackedTab9 make_packed_tab9() {
    PackedTab9 t{};
    for (int n = 0; n < Tab9x9x9::NNZ; ++n) t.v[n] = (uint32_t)Tab9x9x9::I(n) | ((uint32_t)Tab9x9x9::J(n) << 8) | ((uint32_t)Tab9x9x9::K(n) << 16);
    return t;
}
__constant__ PackedTab9 c_tab9 = make_packed_tab9();

constexpr int MAX_NNZ = 256;
constexpr int NG = 3;  // gamma slots in flight

struct StreamParams {
    int64_t N, E;
    int U, D, nnz;
    const int32_t* tab;
    const void* cgw;
    const int32_t* row_ptr;
    const int32_t* ctr;
    const void* gamma;
    const void* Vin;
    const void* Y;
    const void* w0;
    void* Vout;
    const void* gVout;
    void* gVin;
    void* gw0;
    void* gY;
    void* ggamma;
    int gy_tile;        // 1: shuffle-free gY reduction through a shared-memory tile (option tp_stream_gytile)
    int skip_if_baked;  // the three-warp kernel (tp_stream3.cu) was launched for this call: stand down where it works
};

// baked coupling-table structure for a shape (TabNone: none)
template <int D_IN, int D_OUT>
struct BakedTab {
    using type = TabNone;
};
template <>
struct BakedTab<9, 9> {
    using type = Tab9x9x9;
};
template <>
struct BakedTab<4, 4> {
    using type = Tab4x4x4;
};

// row split of the backward (l-aligned for the implicit layer-0 features so that a gw0 row never straddles
// the two warps) and column split of the forward
template <int D_IN, bool IMPLICIT>
struct RowSplit {
    static constexpr int IS = IMPLICIT ? (D_IN == 4 ? 1 : D_IN == 9 ? 4 : D_IN == 16 ? 9 : D_IN / 2) : D_IN / 2;
};

// shared-memory plan (byte offsets), identical on host and device
struct Plan {
    int bars, meta, tab, seg, jperm, jptr, gam, scratch, gyx, ring, stage_bytes, offA, offY, offB, total;
};
template <typename TAct, typename TAcc, int D_IN, int D_OUT, bool IMPLICIT, int MODE>
__host__ __device__ inline Plan make_plan(int U, int D, int NCH, int TE, int NS) {
    Plan p;
    auto up = [](int x) { return (x + 127) & ~127; };
    int o = 0;
    p.bars = o;   o += up((2 * NS + 2 * NG) * 8);
    p.meta = o;   o += up(NG * 8);
    p.tab = o;    o += up(MAX_NNZ * 4);
    p.seg = o;    o += up((D_IN * D_OUT + 1) * 4);
    p.jperm = o;  o += up(MAX_NNZ * 2);
    p.jptr = o;   o += up((D + 1) * 4);
    p.gam = o;    o += up(NG * D * U * (int)sizeof(TAcc));
    p.scratch = o; o += up(NCH * D_IN * D_OUT * 32 * (int)sizeof(TAcc));
    p.gyx = o;    o += (NCH > 1 && MODE == 1 && IMPLICIT) ? up(NCH * TE * D_IN * (int)sizeof(TAcc)) : 0;
    // one stage: [A block: Vin rows | w0 rows] [Y rows] [B block: gVout rows]
    const int n_ir = IMPLICIT ? (D_IN == 1 ? 1 : D_IN == 4 ? 2 : D_IN == 9 ? 3 : D_IN == 16 ? 4 : 5) : 0;
    const int rowA = IMPLICIT ? n_ir * U * (int)sizeof(TAct) : D_IN * U * (int)sizeof(TAct);
    const int rowB = MODE == 1 ? D_OUT * U * (int)sizeof(TAct) : 0;
    p.offA = 0;
    p.offY = up(TE * rowA);
    p.offB = p.offY + (IMPLICIT ? up(TE * ((D_IN + 3) / 4 * 4) * (int)sizeof(TAcc)) : 0);  // Y rows padded to 16 bytes
    p.stage_bytes = p.offB + up(TE * rowB);
    p.ring = o;   o += NS * p.stage_bytes;
    p.total = o;
    return p;
}

// GYT: shuffle-free gY reduction through a shared-memory tile (layer-0 backward, 9 x 9 -> 9, one channel chunk); that build
// only works on the baked table structure and stands down otherwise (the plain build is launched behind it, skip_if_baked)
template <typename TAct, typename TAcc, int D_IN, int D_OUT, bool IMPLICIT, int MODE, int NCH, int TE, int NS, int UT, bool GYT>
__device__ __forceinline__ void tp_stream_body(const StreamParams& p) {
    extern __shared__ __align__(128) uint8_t smem[];
    constexpr int NCW = 2 * NCH;  // consumer warps
    constexpr int T = D_IN * D_OUT;
    constexpr int N_IR = IMPLICIT ? (D_IN == 1 ? 1 : D_IN == 4 ? 2 : D_IN == 9 ? 3 : D_IN == 16 ? 4 : 5) : 0;
    // UT != 0: the channel count is a compile-time constant -> every shared / global offset of the edge loop is an
    // immediate (the first version spent ~2/3 of its instructions on 64-bit index arithmetic with a run-time U)
    const int U = UT ? UT : p.U, D = p.D;
    const Plan pl = make_plan<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE>(U, D, NCH, TE, NS);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + pl.bars);
    int2* s_meta = reinterpret_cast<int2*>(smem + pl.meta);
    uchar4* s_tab = reinterpret_cast<uchar4*>(smem + pl.tab);
    int* s_seg = reinterpret_cast<int*>(smem + pl.seg);
    uint16_t* s_jperm = reinterpret_cast<uint16_t*>(smem + pl.jperm);
    int* s_jptr = reinterpret_cast<int*>(smem + pl.jptr);
    TAcc* s_gam = reinterpret_cast<TAcc*>(smem + pl.gam);
    TAcc* s_scr = reinterpret_cast<TAcc*>(smem + pl.scratch);
    TAcc* s_gyx = reinterpret_cast<TAcc*>(smem + pl.gyx);
    uint8_t* ring = smem + pl.ring;
    const uint32_t bar0 = smem_u32(bars);
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (NS + s); };
    auto gfull_bar = [&](int g) { return bar0 + 8u * (2 * NS + g); };
    auto gempty_bar = [&](int g) { return bar0 + 8u * (2 * NS + NG + g); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nnz = p.nnz;
    if constexpr (D_IN == 9 && D_OUT == 9) {
        if (p.skip_if_baked && nnz == Tab9x9x9::NNZ && p.D == 9) {  // quick stand-down (same test as the full one below)
            int ok = 1;
            for (int n = threadIdx.x; n < Tab9x9x9::NNZ; n += blockDim.x)
                if (((uint32_t)p.tab[3 * n] | ((uint32_t)p.tab[3 * n + 1] << 8) | ((uint32_t)p.tab[3 * n + 2] << 16)) != c_tab9.v[n]) ok = 0;
            if (__syncthreads_and(ok)) return;
        }
    }

    // ---- one-time setup: barriers, tables ----
    if (threadIdx.x == 0) {
        for (int s = 0; s < NS; ++s) {
            mbar_init(full_bar(s), IMPLICIT ? 33 : 1);
            mbar_init(empty_bar(s), NCW);
        }
        for (int g = 0; g < NG; ++g) {
            mbar_init(gfull_bar(g), 1);
            mbar_init(gempty_bar(g), NCW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int n = threadIdx.x; n < nnz; n += blockDim.x)
        s_tab[n] = make_uchar4((unsigned char)p.tab[3 * n], (unsigned char)p.tab[3 * n + 1], (unsigned char)p.tab[3 * n + 2], 0);
    for (int t = threadIdx.x; t <= T; t += blockDim.x) s_seg[t] = -1;
    __syncthreads();
    // segment start of every (i,k) target in the (i,k)-sorted table
    for (int n = threadIdx.x; n < nnz; n += blockDim.x) {
        const int t = s_tab[n].x * D_OUT + s_tab[n].z;
        if (n == 0 || (s_tab[n - 1].x * D_OUT + s_tab[n - 1].z) != t) s_seg[t] = n;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        s_seg[T] = nnz;
        for (int t = T - 1; t >= 0; --t)
            if (s_seg[t] < 0) s_seg[t] = s_seg[t + 1];
    }
    // entries grouped by j (stable: ascending entry id inside a group) for the gM -> ggamma contraction
    if (threadIdx.x < D) {
        int cnt = 0;
        for (int n = 0; n < nnz; ++n) cnt += (s_tab[n].y == threadIdx.x) ? 1 : 0;
        s_jptr[threadIdx.x + 1] = cnt;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        s_jptr[0] = 0;
        for (int j = 0; j < D; ++j) s_jptr[j + 1] += s_jptr[j];
    }
    __syncthreads();
    if (threadIdx.x < D) {
        int pos = s_jptr[threadIdx.x];
        for (int n = 0; n < nnz; ++n)
            if (s_tab[n].y == threadIdx.x) s_jperm[pos++] = (uint16_t)n;
    }
    __syncthreads();

    // ---- does the run-time table have the baked structure?  (then the per-centre contractions are straight-line code) ----
    using TAB = typename BakedTab<D_IN, D_OUT>::type;
    bool baked = false;
    if constexpr (TAB::NNZ > 0) {
        int ok = (nnz == TAB::NNZ && D == TAB::D_ENV) ? 1 : 0;
        for (int n = threadIdx.x; n < TAB::NNZ && ok; n += blockDim.x) {
            const uchar4 t4 = s_tab[n < nnz ? n : 0];
            if (t4.x != TAB::I(n) || t4.y != TAB::J(n) || t4.z != TAB::K(n)) ok = 0;
        }
        baked = __syncthreads_and(ok) != 0 ;
        if (p.skip_if_baked && baked) return;
        if (GYT && !baked) return;
    }

    // ---- this CTA's contiguous range of centres / edges ----
    const int64_t G = gridDim.x, b = blockIdx.x;
    const int64_t c_lo = cut_centre(p.row_ptr, p.ctr, p.N, p.E, b, G);
    const int64_t c_hi = cut_centre(p.row_ptr, p.ctr, p.N, p.E, b + 1, G);
    const int64_t e_lo = p.row_ptr[c_lo], e_hi = p.row_ptr[c_hi];
    const TAct* __restrict__ gA = IMPLICIT ? (const TAct*)p.w0 : (const TAct*)p.Vin;
    const int rowA_el = IMPLICIT ? N_IR * U : D_IN * U;  // elements per edge of the A block
    const int rowB_el = D_OUT * U;
    const uint32_t gam_bytes = (uint32_t)(D * U * sizeof(TAcc));

    if (warp == NCW) {
        // =============================== producer ===============================
        int stage = 0, gslot = 0;
        uint32_t phase = 0, gphase = 0;
        int64_t c_iss = c_lo;  // next centre whose gamma row has not been issued
        // gamma rows run ahead of the edge stages: every non-empty centre beginning before `look_end` is issued.
        // Waiting for a free slot is only allowed for centres that begin inside already issued stages
        // (< issued_end): the consumers can reach those and free a slot.  For look-ahead centres a busy ring
        // just ends the pass (a blocking wait could deadlock when more than NG tiny centres begin in one stage).
        auto issue_gammas = [&](int64_t issued_end, int64_t look_end) {
            while (c_iss < c_hi) {
                const int rb = p.row_ptr[c_iss], re = p.row_ptr[c_iss + 1];
                if (rb >= look_end) break;
                if (re > rb) {
                    if (rb < issued_end) mbar_wait_backoff(gempty_bar(gslot), gphase ^ 1);
                    else if (!mbar_test(gempty_bar(gslot), gphase ^ 1)) break;
                    s_meta[gslot] = make_int2((int)c_iss, re);
                    mbar_expect_tx(gfull_bar(gslot), gam_bytes);
                    bulk_g2s(smem_u32(s_gam + (size_t)gslot * D * U), (const TAcc*)p.gamma + c_iss * D * U, gam_bytes, gfull_bar(gslot));
                    if (++gslot == NG) { gslot = 0; gphase ^= 1; }
                }
                ++c_iss;
            }
        };
        if (lane == 0) issue_gammas(e_lo, e_lo + TE);
        for (int64_t za = e_lo; za < e_hi; za += TE) {
            const int n = (int)((e_hi - za) < TE ? (e_hi - za) : TE);
            if (lane == 0) mbar_wait_backoff(empty_bar(stage), phase ^ 1);
            __syncwarp();
            uint8_t* sb = ring + (size_t)stage * pl.stage_bytes;
            if (lane == 0) {
                const uint32_t bytesA = (uint32_t)(n * rowA_el * sizeof(TAct));
                const uint32_t bytesB = MODE == 1 ? (uint32_t)(n * rowB_el * sizeof(TAct)) : 0u;
                mbar_expect_tx(full_bar(stage), bytesA + bytesB);
                bulk_g2s(smem_u32(sb + pl.offA), gA + za * rowA_el, bytesA, full_bar(stage));
                if (MODE == 1) bulk_g2s(smem_u32(sb + pl.offB), (const TAct*)p.gVout + za * rowB_el, bytesB, full_bar(stage));
            }
            if (IMPLICIT) {
                // Y rows: n * D_IN accumulate-type values, 4-byte aligned only -> element-wise cp.async
                const TAcc* __restrict__ ysrc = (const TAcc*)p.Y + za * D_IN;
                const uint32_t ydst = smem_u32(sb + pl.offY);
                constexpr int YP = (D_IN + 3) / 4 * 4;  // padded row length in shared memory
                for (int e = lane; e < n * D_IN; e += 32) {
                    const int r = e / D_IN, i = e - r * D_IN;
                    if (sizeof(TAcc) == 4) cp_async4(ydst + 4u * (r * YP + i), ysrc + e);
                    else cp_async8(ydst + 8u * (r * YP + i), ysrc + e);
                }
                cp_async_arrive_noinc(full_bar(stage));
            }
            if (lane == 0) issue_gammas(za + n, za + n + TE);
            if (++stage == NS) { stage = 0; phase ^= 1; }
        }
        if (IMPLICIT) asm volatile("cp.async.wait_all;" ::: "memory");
        return;
    }

    // =============================== consumers ===============================
    const int q = warp >> 1, role = warp & 1;  // channel chunk, row/column half
    const int u = q * 32 + lane;
    const bool live = UT ? true : (u < U);
    TAcc* scr = s_scr + (size_t)q * T * 32;
    const TAcc* __restrict__ cgw = (const TAcc*)p.cgw;

    auto run = [&](auto role_tag) {
        constexpr int ROLE = decltype(role_tag)::value;
        constexpr int IS = RowSplit<D_IN, IMPLICIT>::IS;
        constexpr int KS = D_OUT / 2;
        // rows (backward) / columns (forward) owned by this warp
        constexpr int I0 = MODE == 1 ? (ROLE ? IS : 0) : 0;
        constexpr int NI = MODE == 1 ? (ROLE ? D_IN - IS : IS) : D_IN;
        constexpr int K0 = MODE == 0 ? (ROLE ? KS : 0) : 0;
        constexpr int NK = MODE == 0 ? (ROLE ? D_OUT - KS : KS) : D_OUT;
        // M and gM are held as column PAIRS (k, k+1) (+ one single column when NK is odd); fma2 (common.cuh) updates a
        // pair with two FFMAs.
        constexpr int KP = NK / 2, KR = NK % 2;
        [[maybe_unused]] constexpr int YP = (D_IN + 3) / 4 * 4;  // padded Y row in shared memory
        float2 M2[NI][KP > 0 ? KP : 1];
        float Mr[NI];
        float2 gM2[MODE == 1 ? NI : 1][KP > 0 ? KP : 1];
        float gMr[MODE == 1 ? NI : 1];
        int stage = 0, gslot = 0;
        uint32_t phase = 0, gphase = 0;
        int64_t c = -1, c_prev = c_lo - 1;
        int64_t row_end = e_lo;

        auto zero_ggamma = [&](int64_t ca, int64_t cb) {  // centres without edges in (ca, cb): ggamma = 0
            if constexpr (MODE == 1) {
                for (int64_t cc = ca + 1; cc < cb; ++cc)
                    for (int j = role; j < D; j += 2)
                        if (live) ((TAcc*)p.ggamma)[(cc * D + j) * U + u] = TAcc(0);
            }
        };
        auto end_centre = [&]() {
            if constexpr (MODE == 1) {
                // gM -> ggamma[c][j] = sum_nnz cgw * gM[i][k]; both halves meet in the scratch buffer
#pragma unroll
                for (int i = 0; i < NI; ++i) {
#pragma unroll
                    for (int kp = 0; kp < KP; ++kp) {
                        scr[((I0 + i) * D_OUT + 2 * kp) * 32 + lane] = gM2[i][kp].x;
                        scr[((I0 + i) * D_OUT + 2 * kp + 1) * 32 + lane] = gM2[i][kp].y;
                    }
                    if (KR) scr[((I0 + i) * D_OUT + NK - 1) * 32 + lane] = gMr[i];
                }
                named_bar(1 + q, 64);
                if (live) {
                    for (int j = role; j < D; j += 2) {
                        TAcc acc = TAcc(0);
                        for (int n = s_jptr[j]; n < s_jptr[j + 1]; ++n) {
                            const int e = s_jperm[n];
                            const uchar4 t4 = s_tab[e];
                            acc += cgw[(int64_t)e * U + u] * scr[(t4.x * D_OUT + t4.z) * 32 + lane];
                        }
                        ((TAcc*)p.ggamma)[(c * D + j) * U + u] = acc;
                    }
                }
                named_bar(1 + q, 64);  // scratch is reused by the next centre's build
            }
        };
        auto begin_centre = [&]() {
            mbar_wait(gfull_bar(gslot), gphase);
            const int2 mt = s_meta[gslot];
            c = mt.x;
            row_end = mt.y;
            zero_ggamma(c_prev, c);
            c_prev = c;
            const TAcc* __restrict__ gam = s_gam + (size_t)gslot * D * U;
            // every owned M[i][k]: register gather over its table segment, parked in the scratch buffer
            // (table indices are run-time data), then pulled into registers with static indices
            for (int ii = 0; ii < NI; ++ii)
                for (int kk = 0; kk < NK; ++kk) {
                    const int t = (I0 + ii) * D_OUT + (K0 + kk);
                    TAcc acc = TAcc(0);
                    if (live)
                        for (int n = s_seg[t]; n < s_seg[t + 1]; ++n) acc += cgw[(int64_t)n * U + u] * gam[s_tab[n].y * U + u];
                    scr[t * 32 + lane] = acc;
                }
            __syncwarp();
            if (lane == 0) mbar_arrive(gempty_bar(gslot));
            if (++gslot == NG) { gslot = 0; gphase ^= 1; }
#pragma unroll
            for (int i = 0; i < NI; ++i) {
#pragma unroll
                for (int kp = 0; kp < KP; ++kp) {
                    M2[i][kp] = make_float2(scr[((I0 + i) * D_OUT + K0 + 2 * kp) * 32 + lane], scr[((I0 + i) * D_OUT + K0 + 2 * kp + 1) * 32 + lane]);
                    if (MODE == 1) gM2[i][kp] = make_float2(0.f, 0.f);
                }
                if (KR) Mr[i] = scr[((I0 + i) * D_OUT + K0 + NK - 1) * 32 + lane];
                if (MODE == 1) gMr[i] = 0.f;
            }
        };

        // ---- baked-structure versions: every index below is a compile-time constant after unrolling ----
        auto addM = [&](int ii, int kk, float v) {  // M[ii][kk] += v  (ii, kk local to this warp's rows / columns)
            if (kk < 2 * KP) {
                if (kk & 1) M2[ii][kk >> 1].y += v;
                else M2[ii][kk >> 1].x += v;
            } else {
                Mr[ii] += v;
            }
        };
        auto getGM = [&](int ii, int kk) -> float {
            if constexpr (MODE == 1) {
                if (kk < 2 * KP) return (kk & 1) ? gM2[ii][kk >> 1].y : gM2[ii][kk >> 1].x;
                return gMr[ii];
            } else {
                return 0.f;
            }
        };
        int parity_c = 0;  // alternates per centre: two scratch halves -> one barrier per centre
        auto end_centre_baked = [&]() {
            if constexpr (MODE == 1 && TAB::NNZ > 0) {
                // partial ggamma[j] over the table entries whose row i belongs to this warp; the two halves meet in scratch
                float gg[TAB::D_ENV];
#pragma unroll
                for (int j = 0; j < TAB::D_ENV; ++j) gg[j] = 0.f;
#pragma unroll
                for (int n = 0; n < TAB::NNZ; ++n) {
                    const int ti = TAB::I(n), tj = TAB::J(n), tk = TAB::K(n);
                    if (ti >= I0 && ti < I0 + NI) gg[tj] = fmaf(live ? __ldg(cgw + n * U + u) : 0.f, getGM(ti - I0, tk), gg[tj]);
                }
                float* sc = scr + parity_c * (TAB::D_ENV * 32);
                if (ROLE == 1) {
#pragma unroll
                    for (int j = 0; j < TAB::D_ENV; ++j) sc[j * 32 + lane] = gg[j];
                }
                named_bar(1 + q, 64);
                if (ROLE == 0 && live) {
#pragma unroll
                    for (int j = 0; j < TAB::D_ENV; ++j) ((TAcc*)p.ggamma)[(c * D + j) * U + u] = gg[j] + sc[j * 32 + lane];
                }
                parity_c ^= 1;
            }
        };
        auto begin_centre_baked = [&]() {
            if constexpr (TAB::NNZ > 0) {
                mbar_wait(gfull_bar(gslot), gphase);
                const int2 mt = s_meta[gslot];
                c = mt.x;
                row_end = mt.y;
                zero_ggamma(c_prev, c);
                c_prev = c;
                const TAcc* __restrict__ gam = s_gam + (size_t)gslot * D * U + u;
                float g[TAB::D_ENV];
#pragma unroll
                for (int j = 0; j < TAB::D_ENV; ++j) g[j] = live ? gam[j * U] : 0.f;
                __syncwarp();
                if (lane == 0) mbar_arrive(gempty_bar(gslot));
                if (++gslot == NG) { gslot = 0; gphase ^= 1; }
#pragma unroll
                for (int i = 0; i < NI; ++i) {
#pragma unroll
                    for (int kp = 0; kp < KP; ++kp) {
                        M2[i][kp] = make_float2(0.f, 0.f);
                        if (MODE == 1) gM2[i][kp] = make_float2(0.f, 0.f);
                    }
                    if (KR) Mr[i] = 0.f;
                    if (MODE == 1) gMr[i] = 0.f;
                }
#pragma unroll
                for (int n = 0; n < TAB::NNZ; ++n) {
                    const int ti = TAB::I(n), tj = TAB::J(n), tk = TAB::K(n);
                    if (ti >= I0 && ti < I0 + NI && tk >= K0 && tk < K0 + NK) addM(ti - I0, tk - K0, (live ? __ldg(cgw + n * U + u) : 0.f) * g[tj]);
                }
            }
        };

        // running per-lane output pointers (advanced by one edge row per iteration: no 64-bit multiplies in the loop)
        [[maybe_unused]] TAct* __restrict__ vout_p = MODE == 0 ? (TAct*)p.Vout + ((int64_t)e_lo * D_OUT + K0) * U + u : nullptr;
        [[maybe_unused]] TAct* __restrict__ gvin_p = (MODE == 1 && !IMPLICIT) ? (TAct*)p.gVin + ((int64_t)e_lo * D_IN + I0) * U + u : nullptr;
        [[maybe_unused]] TAct* __restrict__ gw0_p = (MODE == 1 && IMPLICIT) ? (TAct*)p.gw0 + (int64_t)e_lo * (N_IR * U) + u : nullptr;
        [[maybe_unused]] float* __restrict__ gy_p = (MODE == 1 && IMPLICIT) ? (float*)p.gY + (int64_t)e_lo * D_IN + I0 : nullptr;
        // shuffle-free gY reduction (layer-0 backward, 9 x 9 -> 9, one channel chunk, baked table): a warp-private tile in the
        // part of the scratch buffer the baked per-centre code does not use ([0, 2 x 9 x 32) floats are its ggamma exchange)
        static_assert(!GYT || (MODE == 1 && IMPLICIT && NCH == 1 && TE == 8 && D_IN == 9 && D_OUT == 9), "gY tile build");
        [[maybe_unused]] float* const gy_tile = GYT ? scr + 2 * 9 * 32 + (ROLE ? TE * RowSplit<D_IN, IMPLICIT>::IS * 16 : 0) : nullptr;
        const int e_lo32 = (int)e_lo, e_hi32 = (int)e_hi;
        int row_end32 = e_lo32;
        for (int za = e_lo32; za < e_hi32; za += TE) {
            const int n = (e_hi32 - za) < TE ? (e_hi32 - za) : TE;
            mbar_wait(full_bar(stage), phase);
            const uint8_t* sb = ring + (size_t)stage * pl.stage_bytes;
            // per-lane bases: element (t, r) of a staged row block is base[(t * ROWS + r) * U]
            const TAct* __restrict__ sA = reinterpret_cast<const TAct*>(sb + pl.offA) + u;
            [[maybe_unused]] const TAcc* __restrict__ sY = reinterpret_cast<const TAcc*>(sb + pl.offY);
            [[maybe_unused]] const TAct* __restrict__ sB = reinterpret_cast<const TAct*>(sb + pl.offB) + u;
            int t = 0;
            while (t < n) {
                if (za + t == row_end32) {  // warp-uniform: first edge of the next non-empty centre
                    if (baked) {
                        if (c >= 0) end_centre_baked();
                        begin_centre_baked();
                    } else {
                        if (c >= 0) end_centre();
                        begin_centre();
                    }
                    row_end32 = (int)row_end;
                }
                // edges of the current centre inside this stage: a branch-free run (unrolled for ILP)
                const int t_end = (row_end32 - za) < n ? (row_end32 - za) : n;
#pragma unroll 2
                for (; t < t_end; ++t) {
                if constexpr (MODE == 0) {
                    // ---------------- forward: Vout[z][K0..][u] = sum_i v[i] M[i][k] ----------------
                    float v[D_IN];
                    if constexpr (IMPLICIT) {
                        float wl[N_IR];
#pragma unroll
                        for (int l = 0; l < N_IR; ++l) wl[l] = live ? to_acc<float>(sA[(t * N_IR + l) * U]) : 0.f;
                        float Yr[YP];
#pragma unroll
                        for (int i4 = 0; i4 < YP / 4; ++i4) {
                            const float4 y4 = *reinterpret_cast<const float4*>(sY + t * YP + 4 * i4);
                            Yr[4 * i4] = y4.x; Yr[4 * i4 + 1] = y4.y; Yr[4 * i4 + 2] = y4.z; Yr[4 * i4 + 3] = y4.w;
                        }
#pragma unroll
                        for (int i = 0; i < D_IN; ++i) v[i] = Yr[i] * wl[sh_l_of(i)];
                    } else {
#pragma unroll
                        for (int i = 0; i < D_IN; ++i) v[i] = live ? to_acc<float>(sA[(t * D_IN + i) * U]) : 0.f;
                    }
                    float2 o2[KP > 0 ? KP : 1];
                    float o_r = 0.f;
#pragma unroll
                    for (int kp = 0; kp < KP; ++kp) o2[kp] = make_float2(0.f, 0.f);
#pragma unroll
                    for (int i = 0; i < D_IN; ++i) {
                        const float2 vv = make_float2(v[i], v[i]);
#pragma unroll
                        for (int kp = 0; kp < KP; ++kp) o2[kp] = fma2(vv, M2[i][kp], o2[kp]);
                        if (KR) o_r = fmaf(v[i], Mr[i], o_r);
                    }
                    if (live) {
#pragma unroll
                        for (int kp = 0; kp < KP; ++kp) {
                            vout_p[(2 * kp) * U] = from_acc<TAct>(o2[kp].x);
                            vout_p[(2 * kp + 1) * U] = from_acc<TAct>(o2[kp].y);
                        }
                        if (KR) vout_p[(NK - 1) * U] = from_acc<TAct>(o_r);
                    }
                    vout_p += D_OUT * U;
                } else {
                    // ---------------- backward ----------------
                    float2 go2[KP > 0 ? KP : 1];
                    float go_r = 0.f;
#pragma unroll
                    for (int kp = 0; kp < KP; ++kp)
                        go2[kp] = live ? make_float2(to_acc<float>(sB[(t * D_OUT + 2 * kp) * U]), to_acc<float>(sB[(t * D_OUT + 2 * kp + 1) * U]))
                                       : make_float2(0.f, 0.f);
                    if (KR) go_r = live ? to_acc<float>(sB[(t * D_OUT + NK - 1) * U]) : 0.f;
                    float v[NI], gin[NI];
                    [[maybe_unused]] float wl[IMPLICIT ? N_IR : 1];
                    [[maybe_unused]] float Yv[IMPLICIT ? NI : 1];
                    if constexpr (IMPLICIT) {
#pragma unroll
                        for (int l = 0; l < N_IR; ++l)
                            if (l * l < I0 + NI && (l + 1) * (l + 1) > I0) wl[l] = live ? to_acc<float>(sA[(t * N_IR + l) * U]) : 0.f;
                        // this warp's rows [I0, I0 + NI) of the padded Y row: aligned 16-byte broadcasts
                        constexpr int A0 = I0 / 4 * 4, A1 = (I0 + NI + 3) / 4 * 4;
                        float Yr[A1 - A0];
#pragma unroll
                        for (int i4 = 0; i4 < (A1 - A0) / 4; ++i4) {
                            const float4 y4 = *reinterpret_cast<const float4*>(sY + t * YP + A0 + 4 * i4);
                            Yr[4 * i4] = y4.x; Yr[4 * i4 + 1] = y4.y; Yr[4 * i4 + 2] = y4.z; Yr[4 * i4 + 3] = y4.w;
                        }
#pragma unroll
                        for (int i = 0; i < NI; ++i) {
                            Yv[i] = Yr[I0 - A0 + i];
                            v[i] = Yv[i] * wl[sh_l_of(I0 + i)];
                        }
                    } else {
#pragma unroll
                        for (int i = 0; i < NI; ++i) v[i] = live ? to_acc<float>(sA[(t * D_IN + I0 + i) * U]) : 0.f;
                    }
#pragma unroll
                    for (int i = 0; i < NI; ++i) {
                        float2 a2 = make_float2(0.f, 0.f);
                        const float2 vv = make_float2(v[i], v[i]);
#pragma unroll
                        for (int kp = 0; kp < KP; ++kp) {
                            a2 = fma2(M2[i][kp], go2[kp], a2);
                            gM2[i][kp] = fma2(vv, go2[kp], gM2[i][kp]);
                        }
                        float s = a2.x + a2.y;
                        if (KR) {
                            s = fmaf(Mr[i], go_r, s);
                            gMr[i] = fmaf(v[i], go_r, gMr[i]);
                        }
                        gin[i] = s;
                    }
                    if constexpr (IMPLICIT) {
                        // Vin[i] = Y[i] w0[l(i)]:  gw0[l] = sum_{i in l} Y[i] gin[i];  gY[i] += sum_u w0[l(i)][u] gin[i]
                        float part[NI];
#pragma unroll
                        for (int l = 0; l < N_IR; ++l) {
                            if (l * l >= I0 && (l + 1) * (l + 1) <= I0 + NI) {  // l owned entirely by this warp
                                float s = 0.f;
#pragma unroll
                                for (int i = l * l; i < (l + 1) * (l + 1); ++i) s = fmaf(Yv[i - I0], gin[i - I0], s);
                                if (live) gw0_p[l * U] = from_acc<TAct>(s);
                            }
                        }
#pragma unroll
                        for (int i = 0; i < NI; ++i) part[i] = wl[sh_l_of(I0 + i)] * gin[i];
                        if constexpr (GYT) {
                            // one xor-16 step (independent shuffles, no chain), lanes 0-15 park the half sums in the tile;
                            // the stage's rows are summed once per stage below, instead of a multi-level shuffle chain
                            // per edge on the edge's critical path.
#pragma unroll
                            for (int i = 0; i < NI; ++i) {
                                const float pr = part[i] + __shfl_xor_sync(0xffffffffu, part[i], 16);
                                if (lane < 16) gy_tile[(t * NI + i) * 16 + lane] = pr;
                            }
                        } else {
                            const float tot = MultiSum<NI>::run(part, lane);
                            const int idx = MultiSum<NI>::idx_of(lane);
                            if (MultiSum<NI>::is_writer(lane) && idx < NI) {
                                if (NCH == 1) atomicAdd(gy_p + idx, tot);  // RED (fire and forget), single writer per address
                                else s_gyx[(q * TE + t) * D_IN + I0 + idx] = tot;
                            }
                        }
                        gw0_p += N_IR * U;
                        gy_p += D_IN;
                    } else {
                        if (live) {
#pragma unroll
                            for (int i = 0; i < NI; ++i) gvin_p[i * U] = from_acc<TAct>(gin[i]);
                        }
                        gvin_p += D_IN * U;
                    }
                }
                }  // run
            }
            if constexpr (GYT) {
                {
                    // row j = (edge j / NI, local row j % NI) of the tile: 16 floats, chunk order rotated per lane so that the
                    // eight lanes of a 128-bit phase hit eight different bank groups; RED, one writer per gY element
                    __syncwarp();
                    for (int j = lane; j < n * NI; j += 32) {
                        const float4* __restrict__ row = reinterpret_cast<const float4*>(gy_tile + j * 16);
                        const int sw = (j >> 1) & 3;
                        const float4 a = row[sw], b4 = row[1 ^ sw], c4 = row[2 ^ sw], d4 = row[3 ^ sw];
                        const float tot = (((a.x + a.y) + (a.z + a.w)) + ((b4.x + b4.y) + (b4.z + b4.w))) + (((c4.x + c4.y) + (c4.z + c4.w)) + ((d4.x + d4.y) + (d4.z + d4.w)));
                        const int tt = j / NI;
                        atomicAdd((float*)p.gY + (int64_t)(za + tt) * D_IN + I0 + (j - tt * NI), tot);
                    }
                }
            }
            if constexpr (NCH > 1 && MODE == 1 && IMPLICIT) {
                // channel chunks of one role meet here: fixed summation order over chunks (deterministic)
                named_bar(3 + role, 32 * NCH);
                if (q == 0) {
                    for (int e = lane; e < n * NI; e += 32) {
                        const int t = e / NI, i = I0 + e % NI;
                        float s = 0.f;
#pragma unroll
                        for (int qq = 0; qq < NCH; ++qq) s += s_gyx[(qq * TE + t) * D_IN + i];
                        atomicAdd((float*)p.gY + (za + t) * D_IN + i, s);
                    }
                }
                named_bar(3 + role, 32 * NCH);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(stage));
            if (++stage == NS) { stage = 0; phase ^= 1; }
        }
        if (c >= 0) {
            if (baked) end_centre_baked();
            else end_centre();
        }
        zero_ggamma(c_prev, c_hi);
    };
    if (role == 0) run(std::integral_constant<int, 0>{});
    else run(std::integral_constant<int, 1>{});
}

// Two entry points over the same body: the plain build keeps the compiler's own register choice (168 for the layer-0
// backward -> 4 CTAs/SM); the gY-tile build needs a few registers more and is capped so that it keeps 4 CTAs/SM
// (a second __launch_bounds__ argument on the plain build changes its allocation: 229 registers with minBlocks = 1).
template <typename TAct, typename TAcc, int D_IN, int D_OUT, bool IMPLICIT, int MODE, int NCH, int TE, int NS, int UT>
__global__ void __launch_bounds__((2 * NCH + 1) * 32) tp_stream_kernel(const StreamParams p) {
    tp_stream_body<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, NCH, TE, NS, UT, false>(p);
}
template <typename TAct, typename TAcc, int D_IN, int D_OUT, bool IMPLICIT, int MODE, int NCH, int TE, int NS, int UT>
__global__ void __launch_bounds__((2 * NCH + 1) * 32, 4) tp_stream_gyt_kernel(const StreamParams p) {
    tp_stream_body<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, NCH, TE, NS, UT, true>(p);
}

template <typename TAct, typename TAcc, int D_IN, int D_OUT, bool IMPLICIT, int MODE, int NCH, int TE, int NS, int UT, bool GYT = false>
int launch_cfg(const StreamParams& p, cudaStream_t st) {
    void (*kern)(const StreamParams);
    if constexpr (GYT) kern = tp_stream_gyt_kernel<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, NCH, TE, NS, UT>;
    else kern = tp_stream_kernel<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, NCH, TE, NS, UT>;
    const Plan pl = make_plan<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE>(p.U, p.D, NCH, TE, NS);
    static int num_sms = 0, max_smem = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    }
    if (pl.total > max_smem) return -1;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, pl.total) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    const int threads = (2 * NCH + 1) * 32;
    int cps = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, kern, threads, pl.total) != cudaSuccess || cps < 1) {
        cudaGetLastError();
        return -1;
    }
    // the 9 -> 1 backward is purely memory-bound: 3 CTAs/SM keep enough bytes in flight.  On an H100 (700 W limit, c2
    // shapes) the cap and the occupancy limit give the same time (0.42 ms per launch), so the cap
    // stays as it is.
    if (D_OUT == 1 && MODE == 1 && cps > 3 && g_ab2_opt_tp_stream_cps == 0) cps = 3;
    // explicit 9 x 9 -> 9 forward (middle layers of models with 3+ layers): capped at 3 CTAs/SM like the 9 -> 1 backward;
    // not measured on an H100 (the benchmark config has no middle layer).  tp_stream_cps overrides both caps.
    if (D_IN == 9 && D_OUT == 9 && MODE == 0 && !IMPLICIT && NCH == 1 && cps > 3 && g_ab2_opt_tp_stream_cps == 0) cps = 3;
    if (g_ab2_opt_tp_stream_cps > 0 && cps > g_ab2_opt_tp_stream_cps) cps = g_ab2_opt_tp_stream_cps;
    int64_t grid = (int64_t)num_sms * cps;
    if (grid > p.N) grid = p.N;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, threads, pl.total, st>>>(p);
    return 0;
}

template <typename TAct, typename TAcc, int D_IN, int D_OUT, bool IMPLICIT, int MODE>
int launch_shape(const StreamParams& p, cudaStream_t st) {
    if (p.U == 32) {
        if constexpr (std::is_same<TAct, float>::value && D_IN == 9 && D_OUT == 9 && IMPLICIT && MODE == 1) {
            if (p.gy_tile && !p.skip_if_baked) {
                // tile build first (works iff the table has the baked structure), then the plain build with the complementary test
                if (launch_cfg<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, 1, 8, 3, 32, true>(p, st) == 0) {
                    StreamParams q = p;
                    q.skip_if_baked = 1;
                    return launch_cfg<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, 1, 8, 3, 32>(q, st);
                }
            }
        }
        return launch_cfg<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, 1, 8, 3, 32>(p, st);
    }
    if (p.U < 32) return launch_cfg<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, 1, 8, 3, 0>(p, st);
    if (p.U == 64) return launch_cfg<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, 2, 8, 2, 64>(p, st);
    if (p.U < 64) return launch_cfg<TAct, TAcc, D_IN, D_OUT, IMPLICIT, MODE, 2, 8, 2, 0>(p, st);
    return -1;
}

// The instantiations are compiled in eight translation units so that a parallel build compiles them side by side
// (about 70 kernels: one translation unit takes about 12 minutes of ptxas time for sm_90a, the slowest of the
// eight under 3 minutes):
// this file (group 0, plus the entry point ab2_tp_stream) and tp_stream_g1.cu .. tp_stream_g7.cu, which define
// AB2_TP_STREAM_GROUP and include this file.  Per storage type TA, the groups are
//   d_in 9 forward | d_in 9 backward with implicit V0 | d_in 9 backward with explicit input (+ 9 -> 1 last layer) | d_in 4.
// Each group is one function: part 0 forward, 1 backward with implicit V0, 2 backward with explicit input.
#ifndef AB2_TP_STREAM_GROUP
#define AB2_TP_STREAM_GROUP 0
#endif
template <typename TA>
int tp_stream_fwd9(const StreamParams& p, bool implicit_v0, cudaStream_t st) {
    return implicit_v0 ? launch_shape<TA, float, 9, 9, true, 0>(p, st) : launch_shape<TA, float, 9, 9, false, 0>(p, st);
}
template <typename TA>
int tp_stream_bwd9_explicit(const StreamParams& p, bool last9, cudaStream_t st) {
    return last9 ? launch_shape<TA, float, 9, 1, false, 1>(p, st) : launch_shape<TA, float, 9, 9, false, 1>(p, st);
}
template <typename TA>
int tp_stream_all4(const StreamParams& p, int part, bool implicit_v0, cudaStream_t st) {
    if (part == 0) return implicit_v0 ? launch_shape<TA, float, 4, 4, true, 0>(p, st) : launch_shape<TA, float, 4, 4, false, 0>(p, st);
    return implicit_v0 ? launch_shape<TA, float, 4, 4, true, 1>(p, st) : launch_shape<TA, float, 4, 4, false, 1>(p, st);
}
}  // namespace

int ab2_tp_stream_group(int group, const void* params, int part, bool implicit_v0, bool last9, cudaStream_t st);
#if AB2_TP_STREAM_GROUP != 0
// group g of storage type TA = (g < 4 ? float : bf16), kind g % 4
static int ab2_tp_stream_group_impl(const void* params, int part, bool implicit_v0, bool last9, cudaStream_t st) {
    using TA = std::conditional<(AB2_TP_STREAM_GROUP < 4), float, bf16>::type;
    const StreamParams& p = *static_cast<const StreamParams*>(params);
    constexpr int kind = AB2_TP_STREAM_GROUP % 4;
    if constexpr (kind == 0) return tp_stream_fwd9<TA>(p, implicit_v0, st);
    else if constexpr (kind == 1) return launch_shape<TA, float, 9, 9, true, 1>(p, st);
    else if constexpr (kind == 2) return tp_stream_bwd9_explicit<TA>(p, last9, st);
    else return tp_stream_all4<TA>(p, part, implicit_v0, st);
}
#define AB2_TP_STREAM_GROUP_SYM_(g) ab2_tp_stream_group##g
#define AB2_TP_STREAM_GROUP_SYM(g) AB2_TP_STREAM_GROUP_SYM_(g)
int AB2_TP_STREAM_GROUP_SYM(AB2_TP_STREAM_GROUP)(const void* params, int part, bool implicit_v0, bool last9, cudaStream_t st) {
    return ab2_tp_stream_group_impl(params, part, implicit_v0, last9, st);
}
#else
int ab2_tp_stream_group1(const void*, int, bool, bool, cudaStream_t);
int ab2_tp_stream_group2(const void*, int, bool, bool, cudaStream_t);
int ab2_tp_stream_group3(const void*, int, bool, bool, cudaStream_t);
int ab2_tp_stream_group4(const void*, int, bool, bool, cudaStream_t);
int ab2_tp_stream_group5(const void*, int, bool, bool, cudaStream_t);
int ab2_tp_stream_group6(const void*, int, bool, bool, cudaStream_t);
int ab2_tp_stream_group7(const void*, int, bool, bool, cudaStream_t);

// launches of group `group` (see above); group 0 (fp32, d_in 9 forward) is instantiated here
int ab2_tp_stream_group(int group, const void* params, int part, bool implicit_v0, bool last9, cudaStream_t st) {
    switch (group) {
        case 0: return tp_stream_fwd9<float>(*static_cast<const StreamParams*>(params), implicit_v0, st);
        case 1: return ab2_tp_stream_group1(params, part, implicit_v0, last9, st);
        case 2: return ab2_tp_stream_group2(params, part, implicit_v0, last9, st);
        case 3: return ab2_tp_stream_group3(params, part, implicit_v0, last9, st);
        case 4: return ab2_tp_stream_group4(params, part, implicit_v0, last9, st);
        case 5: return ab2_tp_stream_group5(params, part, implicit_v0, last9, st);
        case 6: return ab2_tp_stream_group6(params, part, implicit_v0, last9, st);
        case 7: return ab2_tp_stream_group7(params, part, implicit_v0, last9, st);
    }
    return -1;
}

// returns 0 if launched, -1 if (dtype, shape, alignment) has no streaming instantiation
int ab2_tp_stream(int mode, int dtype, int64_t N, int64_t E, int U, int D, int d_in, int d_out, int nnz, const int32_t* tab,
                  const void* cgw, const int32_t* row_ptr, const int32_t* ctr, const void* gamma, const void* Vin, int implicit_v0, const void* Y,
                  const void* w0, int64_t w0_ld, void* Vout, const void* gVout, void* gVin, void* gw0, int64_t gw0_ld, void* gY,
                  void* ggamma, cudaStream_t st) {
    if (!g_ab2_opt_tp_stream || !ctr || dtype == AB2_F64 || nnz > MAX_NNZ || nnz <= 0 || E <= 0 || N <= 0) return -1;
    // last layer of an l_max = 2 model: 9 -> 1 backward (explicit input features), generic per-centre table walk (9 entries)
    const bool last9 = g_ab2_opt_tp_stream_last && mode == 1 && !implicit_v0 && d_in == 9 && d_out == 1 && D == 9;
    if (!last9 && (d_in != d_out || !(d_in == 4 || d_in == 9) || (implicit_v0 && D != d_in))) return -1;
    const int esz = dtype == AB2_F32 ? 4 : 2;
    // bulk copies move whole rows: 16-byte multiples, 16-byte aligned bases, dense rows
    if ((U * esz) % 16 != 0 || (U * 4) % 16 != 0) return -1;
    const int n_ir = d_in == 4 ? 2 : 3;
    if (implicit_v0 && (w0_ld != (int64_t)n_ir * U || (mode == 1 && gw0_ld != (int64_t)n_ir * U))) return -1;
    auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
    if (!al16(gamma) || (implicit_v0 ? !al16(w0) : !al16(Vin)) || (mode == 1 && !al16(gVout))) return -1;
    StreamParams p;
    p.N = N; p.E = E; p.U = U; p.D = D; p.nnz = nnz; p.tab = tab; p.cgw = cgw; p.row_ptr = row_ptr; p.ctr = ctr; p.gamma = gamma;
    p.Vin = Vin; p.Y = Y; p.w0 = w0; p.Vout = Vout; p.gVout = gVout; p.gVin = gVin; p.gw0 = gw0; p.gY = gY; p.ggamma = ggamma;
    // layer-0 backward at the l_max = 2 shape: three consumer warps per centre stream (tp_stream3.cu).  That kernel only
    // works on the baked table structure and checks it on the device; the two-warp kernel below runs with the
    // complementary test, so exactly one of the two launches does the work (no host-side look at device data).
    p.skip_if_baked = 0;
    p.gy_tile = g_ab2_opt_tp_stream_gytile;
    if (mode == 1 && implicit_v0 && dtype == AB2_F32 && d_in == 9 && D == 9 && U == 32 && nnz == Tab9x9x9::NNZ && E < ((int64_t)1 << 31) &&
        ab2_tp_stream3_bwd(N, E, tab, cgw, row_ptr, ctr, gamma, Y, w0, gVout, gw0, gY, ggamma, st) == 0)
        p.skip_if_baked = 1;
    const int base = dtype == AB2_F32 ? 0 : 4;
    if (last9) {
        p.skip_if_baked = 0;
        p.gy_tile = 0;
        return ab2_tp_stream_group(base + 2, &p, 2, false, true, st);
    }
    if (d_in == 4) return ab2_tp_stream_group(base + 3, &p, mode, implicit_v0, false, st);
    if (mode == 0) return ab2_tp_stream_group(base + 0, &p, 0, implicit_v0, false, st);
    return ab2_tp_stream_group(base + (implicit_v0 ? 1 : 2), &p, 1, implicit_v0, false, st);
}
#endif

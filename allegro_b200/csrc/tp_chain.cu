// Composed tensor product of a two-layer l_max = 2 model (ab2_tp_chain_fwd / ab2_tp_chain_bwd): the layer-1 tensor
// features V_1[E][9][U] and their gradient are never formed.
//
// Reference semantics: the two Contracter calls of Allegro_Module.forward (allegro/nn/_allegro.py:237-301) for
// num_layers = 2, where nothing touches the tensor track between the layers:  V_1 = tp0(V_0, Gamma_0),  s_1 = V_1[0],
// s_2 = tp1(V_1, Gamma_1)[0],  with V_0 = Y (x) w0 implicit (tensorembed.py:95).
//
// The algebra (per channel u, dropped below).  Both products are linear in their first operand and their coupling
// depends on the centre only, so with v0[i] = Y[i] w0[l(i)]:
//   M0_c[i][k] = sum_{(i,j,k) in tab0} cgw0 Gamma0_c[j],   M1_c[k] = sum_{(k,j,0) in tab1} cgw1 Gamma1_c[j]
//   s_1 = sum_i A_c[i] v0[i],   A_c[i] = M0_c[i][0]
//   s_2 = sum_i B_c[i] v0[i],   B_c[i] = sum_k M0_c[i][k] M1_c[k]
// and the adjoint, given g1 = d/ds_1 and g2 = d/ds_2 per edge:
//   gv0[i] = A_c[i] g1 + B_c[i] g2         -> gw0[l] = sum_{i in l} Y[i] gv0[i],  gY[i] += sum_u w0[l(i)] gv0[i]
//   G_c[i] = sum_{z in c} g2 v0[i],  H_c[i] = sum_{z in c} g1 v0[i]
//   gGamma1_c[j] = sum_{(k,j,0) in tab1} cgw1 sum_i M0_c[i][k] G_c[i]
//   gGamma0_c[j] = sum_{(i,j,k) in tab0} cgw0 (delta_k0 H_c[i] + M1_c[k] G_c[i])
// A_c and B_c are straight-line code over the baked table structures (tp_tables_generated.cuh): the 9 x 9 matrix M0 is
// never built.  Per edge the kernels read Y, w0 and the compact [E][U] scalars; V_1 is 1152 B per edge at U = 32.
//
// Staging as in tp_stream.cu: CTA b owns a contiguous edge range cut at centre boundaries.  One producer warp brings the
// w0 (and g1 / g2) rows in with 1-D bulk copies and the Y rows with cp.async, in stages of TE edges, and the Gamma rows
// of each non-empty centre ahead of the edges into NG slots.  One consumer warp (lane = channel, U / 32 channel chunks
// per lane) walks the edges.  A centre keeps its Gamma slot until it ends, so the backward reads the rows there again
// for its once-per-centre gGamma.  Every sum runs in a fixed order and gGamma is written once per centre (empty
// centres: zero), so the results do not depend on the launch.
#include "common.cuh"
#include "stream_common.cuh"
#include "tp_tables_generated.cuh"

namespace {

using TAB0 = Tab9x9x9;
using TAB1 = Tab9x9x1;
constexpr int CD = 9, CN_IR = 3, CYP = 12;  // components, irreps, padded Y row
constexpr int CTE = 8, CNS = 3, CNG = 3;     // edges per stage, stages, Gamma slots

enum { CH_FWD_A = 0, CH_FWD_B = 1, CH_BWD_LAST = 2, CH_BWD_FIRST = 3 };

struct ChainParams {
    int64_t N, E;
    const int32_t* row_ptr;
    const int32_t* ctr;
    const float* cgw0;
    const float* cgw1;
    const float* gamma0;
    const float* gamma1;
    const float* Y;
    const float* w0;
    const float* g1;
    const float* g2;
    float* s;
    float* gw0;
    float* gY;
    float* ggamma;
};

// per-edge row blocks of a stage: w0 [3U], then the gradient rows (last-layer backward: g2; first-layer backward: g1, g2)
template <int MODE>
struct ChainShape {
    static constexpr int NGAM = (MODE == CH_FWD_B || MODE == CH_BWD_FIRST) ? 2 : 1;  // Gamma rows per centre
    static constexpr int NGRAD = MODE == CH_BWD_LAST ? 1 : MODE == CH_BWD_FIRST ? 2 : 0;
};

struct ChainPlan {
    int bars, meta, gam, ring, offY, offG, stage_bytes, total;
};
template <int MODE>
__host__ __device__ inline ChainPlan chain_plan(int U) {
    auto up = [](int x) { return (x + 127) & ~127; };
    ChainPlan p;
    int o = 0;
    p.bars = o;  o += up((2 * CNS + 2 * CNG) * 8);
    p.meta = o;  o += up(CNG * 8);
    p.gam = o;   o += CNG * ChainShape<MODE>::NGAM * CD * U * 4;
    p.offY = CTE * CN_IR * U * 4;
    p.offG = p.offY + CTE * CYP * 4;
    p.stage_bytes = up(p.offG + ChainShape<MODE>::NGRAD * CTE * U * 4);
    p.ring = o;  o += CNS * p.stage_bytes;
    p.total = o;
    return p;
}

template <int MODE, int NCH>
__global__ void __launch_bounds__(64) tp_chain_kernel(const ChainParams p) {
    constexpr int U = 32 * NCH;
    constexpr int NGAM = ChainShape<MODE>::NGAM, NGRAD = ChainShape<MODE>::NGRAD;
    constexpr bool BWD = MODE >= CH_BWD_LAST;
    extern __shared__ __align__(128) uint8_t smem[];
    const ChainPlan pl = chain_plan<MODE>(U);
    int2* s_meta = reinterpret_cast<int2*>(smem + pl.meta);
    float* s_gam = reinterpret_cast<float*>(smem + pl.gam);
    uint8_t* ring = smem + pl.ring;
    const uint32_t bar0 = smem_u32(smem + pl.bars);
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (CNS + s); };
    auto gfull_bar = [&](int g) { return bar0 + 8u * (2 * CNS + g); };
    auto gempty_bar = [&](int g) { return bar0 + 8u * (2 * CNS + CNG + g); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < CNS; ++s) {
            mbar_init(full_bar(s), 33);  // expect_tx arrive of lane 0 + 32 cp.async (noinc) arrivals
            mbar_init(empty_bar(s), 1);
        }
        for (int g = 0; g < CNG; ++g) {
            mbar_init(gfull_bar(g), 1);
            mbar_init(gempty_bar(g), 1);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int64_t G = gridDim.x, b = blockIdx.x;
    const int64_t c_lo = cut_centre(p.row_ptr, p.ctr, p.N, p.E, b, G);
    const int64_t c_hi = cut_centre(p.row_ptr, p.ctr, p.N, p.E, b + 1, G);
    const int e_lo = p.row_ptr[c_lo], e_hi = p.row_ptr[c_hi];
    const uint32_t gam_bytes = (uint32_t)(CD * U * 4);

    if (warp == 1) {
        // =============================== producer ===============================
        int stage = 0, gslot = 0;
        uint32_t phase = 0, gphase = 0;
        int64_t c_iss = c_lo;  // next centre whose Gamma rows have not been issued
        // Gamma rows run ahead of the edge stages (tp_stream.cu): a blocking wait for a free slot only for centres that
        // begin inside already issued stages, whose predecessors the consumer can finish; look-ahead centres wait for a
        // later pass when the slots are busy.
        auto issue_gammas = [&](int64_t issued_end, int64_t look_end) {
            while (c_iss < c_hi) {
                const int rb = p.row_ptr[c_iss], re = p.row_ptr[c_iss + 1];
                if (rb >= look_end) break;
                if (re > rb) {
                    if (rb < issued_end) mbar_wait_backoff(gempty_bar(gslot), gphase ^ 1);
                    else if (!mbar_test(gempty_bar(gslot), gphase ^ 1)) break;
                    s_meta[gslot] = make_int2((int)c_iss, re);
                    mbar_expect_tx(gfull_bar(gslot), NGAM * gam_bytes);
                    float* dst = s_gam + (size_t)gslot * NGAM * CD * U;
                    bulk_g2s(smem_u32(dst), p.gamma0 + c_iss * CD * U, gam_bytes, gfull_bar(gslot));
                    if (NGAM == 2) bulk_g2s(smem_u32(dst + CD * U), p.gamma1 + c_iss * CD * U, gam_bytes, gfull_bar(gslot));
                    if (++gslot == CNG) { gslot = 0; gphase ^= 1; }
                }
                ++c_iss;
            }
        };
        if (lane == 0) issue_gammas(e_lo, e_lo + CTE);
        for (int za = e_lo; za < e_hi; za += CTE) {
            const int n = (e_hi - za) < CTE ? (e_hi - za) : CTE;
            if (lane == 0) mbar_wait_backoff(empty_bar(stage), phase ^ 1);
            __syncwarp();
            uint8_t* sb = ring + (size_t)stage * pl.stage_bytes;
            if (lane == 0) {
                const uint32_t bw = (uint32_t)(n * CN_IR * U * 4), bg = (uint32_t)(n * U * 4);
                mbar_expect_tx(full_bar(stage), bw + NGRAD * bg);
                bulk_g2s(smem_u32(sb), p.w0 + (int64_t)za * CN_IR * U, bw, full_bar(stage));
                if (MODE == CH_BWD_LAST) bulk_g2s(smem_u32(sb + pl.offG), p.g2 + (int64_t)za * U, bg, full_bar(stage));
                if (MODE == CH_BWD_FIRST) {
                    bulk_g2s(smem_u32(sb + pl.offG), p.g1 + (int64_t)za * U, bg, full_bar(stage));
                    bulk_g2s(smem_u32(sb + pl.offG + CTE * U * 4), p.g2 + (int64_t)za * U, bg, full_bar(stage));
                }
            }
            // Y rows: 36 B each, 4-byte aligned only -> element-wise cp.async into 48-byte rows
            const float* __restrict__ ysrc = p.Y + (int64_t)za * CD;
            const uint32_t ydst = smem_u32(sb + pl.offY);
            for (int e = lane; e < n * CD; e += 32) {
                const int r = e / CD, i = e - r * CD;
                cp_async4(ydst + 4u * (r * CYP + i), ysrc + e);
            }
            cp_async_arrive_noinc(full_bar(stage));
            if (lane == 0) issue_gammas(za + n, za + n + CTE);
            if (++stage == CNS) { stage = 0; phase ^= 1; }
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        return;
    }

    // =============================== consumer ===============================
    // per chunk q (channel u = 32 q + lane): Q = A (layer-0 forward, first-layer backward) or B (layer-1 forward) and,
    // in the first-layer backward, B as well; G / H the per-centre sums of the backward
    float Q[NCH][CD];
    [[maybe_unused]] float Bm[MODE == CH_BWD_FIRST ? NCH : 1][CD];
    [[maybe_unused]] float Gs[BWD ? NCH : 1][CD];
    [[maybe_unused]] float Hs[MODE == CH_BWD_FIRST ? NCH : 1][CD];
    int stage = 0, gslot = 0;
    uint32_t phase = 0, gphase = 0;
    int64_t c = -1, c_prev = c_lo - 1;
    int row_end = e_lo;
    const float* gam = s_gam;  // the current centre's slot

    auto zero_ggamma = [&](int64_t ca, int64_t cb) {  // centres without edges in (ca, cb): gGamma = 0
        if constexpr (BWD) {
            for (int64_t cc = ca + 1; cc < cb; ++cc)
                for (int j = 0; j < CD; ++j)
#pragma unroll
                    for (int q = 0; q < NCH; ++q) p.ggamma[(cc * CD + j) * U + q * 32 + lane] = 0.f;
        }
    };
    // M1_c[k] of chunk q from the slot's Gamma_1 row
    auto build_m1 = [&](int q, float (&m1)[CD]) {
        const int u = q * 32 + lane;
#pragma unroll
        for (int k = 0; k < CD; ++k) m1[k] = 0.f;
#pragma unroll
        for (int n = 0; n < TAB1::NNZ; ++n)
            m1[TAB1::I(n)] = fmaf(__ldg(p.cgw1 + n * U + u), gam[CD * U + TAB1::J(n) * U + u], m1[TAB1::I(n)]);
    };
    auto begin_centre = [&]() {
        mbar_wait(gfull_bar(gslot), gphase);
        const int2 mt = s_meta[gslot];
        c = mt.x;
        row_end = mt.y;
        zero_ggamma(c_prev, c);
        c_prev = c;
        gam = s_gam + (size_t)gslot * NGAM * CD * U;
#pragma unroll
        for (int q = 0; q < NCH; ++q) {
            const int u = q * 32 + lane;
            float g0[CD];
#pragma unroll
            for (int j = 0; j < CD; ++j) g0[j] = gam[j * U + u];
            if constexpr (MODE == CH_FWD_A || MODE == CH_BWD_FIRST) {
                // A[i] = M0[i][0]
#pragma unroll
                for (int i = 0; i < CD; ++i) Q[q][i] = 0.f;
#pragma unroll
                for (int n = 0; n < TAB0::NNZ; ++n)
                    if (TAB0::K(n) == 0) Q[q][TAB0::I(n)] = fmaf(__ldg(p.cgw0 + n * U + u), g0[TAB0::J(n)], Q[q][TAB0::I(n)]);
            }
            if constexpr (MODE == CH_FWD_B || MODE == CH_BWD_FIRST) {
                // B[i] = sum_k M0[i][k] M1[k]
                float m1[CD];
                build_m1(q, m1);
                float bb[CD];
#pragma unroll
                for (int i = 0; i < CD; ++i) bb[i] = 0.f;
#pragma unroll
                for (int n = 0; n < TAB0::NNZ; ++n)
                    bb[TAB0::I(n)] = fmaf(__ldg(p.cgw0 + n * U + u) * g0[TAB0::J(n)], m1[TAB0::K(n)], bb[TAB0::I(n)]);
#pragma unroll
                for (int i = 0; i < CD; ++i) {
                    if constexpr (MODE == CH_FWD_B) Q[q][i] = bb[i];
                    else Bm[q][i] = bb[i];
                }
            }
            if constexpr (BWD) {
#pragma unroll
                for (int i = 0; i < CD; ++i) Gs[q][i] = 0.f;
            }
            if constexpr (MODE == CH_BWD_FIRST) {
#pragma unroll
                for (int i = 0; i < CD; ++i) Hs[q][i] = 0.f;
            }
        }
    };
    auto end_centre = [&]() {
        if constexpr (MODE == CH_BWD_LAST) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
                const int u = q * 32 + lane;
                // gM1[k] = sum_i M0[i][k] G[i];  gGamma1[j] = sum_{(k,j,0)} cgw1 gM1[k]
                float gm1[CD], gg[CD];
#pragma unroll
                for (int k = 0; k < CD; ++k) gm1[k] = gg[k] = 0.f;
#pragma unroll
                for (int n = 0; n < TAB0::NNZ; ++n)
                    gm1[TAB0::K(n)] = fmaf(__ldg(p.cgw0 + n * U + u) * gam[TAB0::J(n) * U + u], Gs[q][TAB0::I(n)], gm1[TAB0::K(n)]);
#pragma unroll
                for (int n = 0; n < TAB1::NNZ; ++n) gg[TAB1::J(n)] = fmaf(__ldg(p.cgw1 + n * U + u), gm1[TAB1::I(n)], gg[TAB1::J(n)]);
#pragma unroll
                for (int j = 0; j < CD; ++j) p.ggamma[(c * CD + j) * U + u] = gg[j];
            }
        }
        if constexpr (MODE == CH_BWD_FIRST) {
#pragma unroll
            for (int q = 0; q < NCH; ++q) {
                const int u = q * 32 + lane;
                // gGamma0[j] = sum_{(i,j,k)} cgw0 (delta_k0 H[i] + M1[k] G[i])
                float m1[CD], gg[CD];
                build_m1(q, m1);
#pragma unroll
                for (int j = 0; j < CD; ++j) gg[j] = 0.f;
#pragma unroll
                for (int n = 0; n < TAB0::NNZ; ++n) {
                    const int i = TAB0::I(n), k = TAB0::K(n);
                    const float t = k == 0 ? fmaf(m1[0], Gs[q][i], Hs[q][i]) : m1[k] * Gs[q][i];
                    gg[TAB0::J(n)] = fmaf(__ldg(p.cgw0 + n * U + u), t, gg[TAB0::J(n)]);
                }
#pragma unroll
                for (int j = 0; j < CD; ++j) p.ggamma[(c * CD + j) * U + u] = gg[j];
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(gempty_bar(gslot));
        if (++gslot == CNG) { gslot = 0; gphase ^= 1; }
    };

    // running per-lane output pointers (one edge row per iteration)
    [[maybe_unused]] float* __restrict__ s_p = BWD ? nullptr : p.s + (int64_t)e_lo * U + lane;
    [[maybe_unused]] float* __restrict__ gw0_p = MODE == CH_BWD_FIRST ? p.gw0 + (int64_t)e_lo * CN_IR * U + lane : nullptr;
    [[maybe_unused]] float* __restrict__ gy_p = MODE == CH_BWD_FIRST ? p.gY + (int64_t)e_lo * CD : nullptr;
    for (int za = e_lo; za < e_hi; za += CTE) {
        const int n = (e_hi - za) < CTE ? (e_hi - za) : CTE;
        mbar_wait(full_bar(stage), phase);
        const uint8_t* sb = ring + (size_t)stage * pl.stage_bytes;
        const float* __restrict__ sW = reinterpret_cast<const float*>(sb) + lane;
        const float* __restrict__ sY = reinterpret_cast<const float*>(sb + pl.offY);
        [[maybe_unused]] const float* __restrict__ sG = reinterpret_cast<const float*>(sb + pl.offG) + lane;
        int t = 0;
        while (t < n) {
            if (za + t == row_end) {  // warp-uniform: first edge of the next non-empty centre
                if (c >= 0) end_centre();
                begin_centre();
            }
            const int t_end = (row_end - za) < n ? (row_end - za) : n;
#pragma unroll 2
            for (; t < t_end; ++t) {
                float Yr[CYP];
#pragma unroll
                for (int i4 = 0; i4 < CYP / 4; ++i4) {
                    const float4 y4 = *reinterpret_cast<const float4*>(sY + t * CYP + 4 * i4);
                    Yr[4 * i4] = y4.x; Yr[4 * i4 + 1] = y4.y; Yr[4 * i4 + 2] = y4.z; Yr[4 * i4 + 3] = y4.w;
                }
                if constexpr (!BWD) {
                    // s = sum_l w0[l] sum_{i in l} Q[i] Y[i]
#pragma unroll
                    for (int q = 0; q < NCH; ++q) {
                        float acc = 0.f;
#pragma unroll
                        for (int l = 0; l < CN_IR; ++l) {
                            float pl_ = 0.f;
#pragma unroll
                            for (int i = l * l; i < (l + 1) * (l + 1); ++i) pl_ = fmaf(Q[q][i], Yr[i], pl_);
                            acc = fmaf(sW[(t * CN_IR + l) * U + q * 32], pl_, acc);
                        }
                        s_p[q * 32] = acc;
                    }
                    s_p += U;
                } else if constexpr (MODE == CH_BWD_LAST) {
                    // G[i] += g2 w0[l(i)] Y[i]
#pragma unroll
                    for (int q = 0; q < NCH; ++q) {
                        const float g2 = sG[t * U + q * 32];
#pragma unroll
                        for (int l = 0; l < CN_IR; ++l) {
                            const float gw = g2 * sW[(t * CN_IR + l) * U + q * 32];
#pragma unroll
                            for (int i = l * l; i < (l + 1) * (l + 1); ++i) Gs[q][i] = fmaf(gw, Yr[i], Gs[q][i]);
                        }
                    }
                } else {
                    float part[CD];
#pragma unroll
                    for (int i = 0; i < CD; ++i) part[i] = 0.f;
#pragma unroll
                    for (int q = 0; q < NCH; ++q) {
                        const float g1 = sG[t * U + q * 32], g2 = sG[CTE * U + t * U + q * 32];
#pragma unroll
                        for (int l = 0; l < CN_IR; ++l) {
                            const float wl = sW[(t * CN_IR + l) * U + q * 32];
                            const float a1 = g1 * wl, a2 = g2 * wl;
                            float gwl = 0.f;
#pragma unroll
                            for (int i = l * l; i < (l + 1) * (l + 1); ++i) {
                                const float gv = fmaf(Q[q][i], g1, Bm[q][i] * g2);  // gv0[i]
                                gwl = fmaf(Yr[i], gv, gwl);
                                part[i] = fmaf(wl, gv, part[i]);
                                Hs[q][i] = fmaf(a1, Yr[i], Hs[q][i]);
                                Gs[q][i] = fmaf(a2, Yr[i], Gs[q][i]);
                            }
                            gw0_p[l * U + q * 32] = gwl;
                        }
                    }
                    gw0_p += CN_IR * U;
                    // gY[z][i] += sum over channels: one multi-value butterfly over components 0..7, one over component 8;
                    // one RED per (z, i), a single writer per address
                    float v8[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) v8[i] = part[i];
                    const float tot = MultiSum<8>::run(v8, lane);
                    if (MultiSum<8>::is_writer(lane)) atomicAdd(gy_p + MultiSum<8>::idx_of(lane), tot);
                    const float t8 = warp_sum(part[8]);
                    if (lane == 0) atomicAdd(gy_p + 8, t8);
                    gy_p += CD;
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(stage));
        if (++stage == CNS) { stage = 0; phase ^= 1; }
    }
    if (c >= 0) end_centre();
    zero_ggamma(c_prev, c_hi);
}

template <int MODE, int NCH>
int chain_launch(const ChainParams& p, cudaStream_t st) {
    auto kern = tp_chain_kernel<MODE, NCH>;
    const ChainPlan pl = chain_plan<MODE>(32 * NCH);
    static int num_sms = 0, max_smem = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    }
    if (pl.total > max_smem) return AB2_NOT_ELIGIBLE;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, pl.total) != cudaSuccess) {
        cudaGetLastError();
        return AB2_NOT_ELIGIBLE;
    }
    int cps = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cps, kern, 64, pl.total) != cudaSuccess || cps < 1) {
        cudaGetLastError();
        return AB2_NOT_ELIGIBLE;
    }
    int64_t grid = (int64_t)num_sms * cps;
    if (grid > p.N) grid = p.N;
    if (grid < 1) grid = 1;
    kern<<<(unsigned)grid, 64, pl.total, st>>>(p);
    return 0;
}

template <int MODE>
int chain_dispatch(int U, const ChainParams& p, cudaStream_t st) {
    return U == 32 ? chain_launch<MODE, 1>(p, st) : chain_launch<MODE, 2>(p, st);
}

bool chain_args_ok(int dtype, int64_t N, int64_t E, int U, const void* const* rows, int n_rows) {
    if (dtype != AB2_F32 || !(U == 32 || U == 64) || N <= 0 || E <= 0 || E >= ((int64_t)1 << 31)) return false;
    for (int r = 0; r < n_rows; ++r)  // bulk-copied bases
        if (!rows[r] || (reinterpret_cast<uintptr_t>(rows[r]) & 15) != 0) return false;
    return true;
}

}  // namespace

extern "C" int ab2_tp_chain_fwd(int dtype, int last, int64_t N, int64_t E, int U, const int32_t* row_ptr, const int32_t* ctr,
                                const void* cgw0, const void* cgw1, const void* gamma0, const void* gamma1, const void* Y,
                                const void* w0, void* s, void* stream) {
    const void* rows[3] = {gamma0, last ? gamma1 : gamma0, w0};
    if (!chain_args_ok(dtype, N, E, U, rows, 3)) return AB2_NOT_ELIGIBLE;
    AB2_CHECK_ARG(row_ptr && ctr && cgw0 && (!last || cgw1) && Y && s, "null pointer");
    ChainParams p{};
    p.N = N; p.E = E; p.row_ptr = row_ptr; p.ctr = ctr; p.cgw0 = (const float*)cgw0; p.cgw1 = (const float*)cgw1;
    p.gamma0 = (const float*)gamma0; p.gamma1 = (const float*)gamma1; p.Y = (const float*)Y; p.w0 = (const float*)w0; p.s = (float*)s;
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = last ? chain_dispatch<CH_FWD_B>(U, p, st) : chain_dispatch<CH_FWD_A>(U, p, st);
    if (rc != 0) return rc;
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_tp_chain_bwd(int dtype, int first, int64_t N, int64_t E, int U, const int32_t* row_ptr, const int32_t* ctr,
                                const void* cgw0, const void* cgw1, const void* gamma0, const void* gamma1, const void* Y,
                                const void* w0, const void* g1, const void* g2, void* gw0, void* gY, void* ggamma, void* stream) {
    const void* rows[5] = {gamma0, first ? gamma1 : gamma0, w0, first ? g1 : g2, g2};
    if (!chain_args_ok(dtype, N, E, U, rows, 5)) return AB2_NOT_ELIGIBLE;
    AB2_CHECK_ARG(row_ptr && ctr && cgw0 && cgw1 && Y && ggamma && (!first || (gw0 && gY)), "null pointer");
    ChainParams p{};
    p.N = N; p.E = E; p.row_ptr = row_ptr; p.ctr = ctr; p.cgw0 = (const float*)cgw0; p.cgw1 = (const float*)cgw1;
    p.gamma0 = (const float*)gamma0; p.gamma1 = (const float*)gamma1; p.Y = (const float*)Y; p.w0 = (const float*)w0;
    p.g1 = (const float*)g1; p.g2 = (const float*)g2; p.gw0 = (float*)gw0; p.gY = (float*)gY; p.ggamma = (float*)ggamma;
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = first ? chain_dispatch<CH_BWD_FIRST>(U, p, st) : chain_dispatch<CH_BWD_LAST>(U, p, st);
    if (rc != 0) return rc;
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// Layer-0 tensor-product backward, THREE consumer warps per 32-channel centre stream.
//
// Same semantics, data layout and TMA-staged pipeline as tp_stream_kernel<9, 9, implicit, bwd> (tp_stream.cu; reference:
// Contracter._contract, allegro/nn/_strided/_contract.py:213-251, its two backward products _flashallegro.py:347-360,
// and the V0 = Y (x) w0 embedding of tensorembed.py:95 folded in), specialised to the l_max = 2 layer-0 shape
// (d_in = d_env = d_out = 9, fp32, U = 32) with the baked 83-entry coupling-table structure.
//
// Why.  The two-warp kernel is latency-bound, not throughput-bound (no pipe saturated, stalls on fixed-latency
// dependencies and the shared-memory scoreboard): 168 registers -> 4 CTAs/SM -> only 8 consumer warps per SM
// (2 per sub-partition) to cover the LDS -> FMA chain -> shuffle-reduction latency of an edge.  Splitting the
// coupling matrix M_c and its gradient gM_c over THREE row groups {1,2,3} | {4,5,6} | {0,7,8} needs 27 + 27 resident values
// per lane instead of 45 + 45 -> <= 128 registers -> 4 CTAs/SM x 3 = 12 consumer warps per SM at the same shared-memory
// footprint.  The l = 2 block of gw0 straddles two warps (rows 4-6 | 7-8): warp C parks its partial in a per-stage slot
// (published on an mbarrier, the ring's own flow control makes the slot safe to reuse), warp B adds its own and stores.
// Everything stays single-writer and fixed-order (deterministic); gVout / w0 / Y are read once, ggamma written once.
#include <type_traits>

#include "common.cuh"
#include "tp_fast.cuh"
#include "tp_tables_generated.cuh"
#include "stream_common.cuh"

int g_ab2_opt_tp_stream3 = 1;  // 1 (default): three-warp backward where eligible, 0: two-warp tp_stream kernel
// stage knock-outs for tools/time_tp3.py (results are WRONG when non-zero): bit0 consumers skip the edge arithmetic,
// bit1 no gY reduction / RED, bit2 no RED only, bit3 producer polls without back-off, bit4 no Y copies, bit5 no per-centre work,
// bit6 compute only (no bulk copies); bit8 selects the unroll-2 build instead of the default unroll-1 (results stay right)
int g_ab2_opt_tp_stream3_debug = 0;

namespace {

constexpr int U3 = 32, D3 = 9, NIR3 = 3, TE3 = 8, NS3 = 3, NG3 = 3;
constexpr int YP3 = 12;  // Y row padded to 48 bytes in shared memory
using TAB3 = Tab9x9x9;

struct Params3 {
    int64_t N, E;
    const int32_t* tab;
    const float* cgw;
    const int32_t* row_ptr;
    const int32_t* ctr;
    const float* gamma;
    const float* Y;
    const float* w0;
    const float* gVout;
    float* gw0;
    float* gY;
    float* ggamma;
    int debug;
};

// shared-memory plan (bytes)
constexpr int OFF_BARS = 0;                                  // full[NS], empty[NS], gfull[NG], gempty[NG], xfull[NS]
constexpr int OFF_META = 128;                                // int2[NG]
constexpr int OFF_GAM = 256;                                 // NG x 9 x 32 floats
constexpr int OFF_XG = OFF_GAM + NG3 * D3 * U3 * 4;          // ggamma partials: 2 parities x 2 senders x 9 x 32 floats
constexpr int OFF_XW = OFF_XG + 2 * 2 * D3 * U3 * 4;         // gw0[l=2] partial of warp C: NS x TE x 32 floats
constexpr int OFF_XB = OFF_XW + NS3 * TE3 * U3 * 4;          // gw0[l=2] partial of warp B (private): TE x 32 floats
constexpr int OFF_TY = OFF_XB + TE3 * U3 * 4;                // gY partials (lanes 0-15 after one xor-16 step): 3 warps x TE x 3 x 16 floats
constexpr int OFF_RING = OFF_TY + 3 * TE3 * 3 * 16 * 4;
constexpr int ST_A = 0;                                      // w0 rows   TE x 3 x 32 floats
constexpr int ST_Y = TE3 * NIR3 * U3 * 4;                    // Y rows    TE x 12 floats
constexpr int ST_B = ST_Y + TE3 * YP3 * 4;                   // gVout rows TE x 9 x 32 floats
constexpr int STAGE_BYTES = ST_B + TE3 * D3 * U3 * 4;
constexpr int SMEM3 = OFF_RING + NS3 * STAGE_BYTES;
static_assert(OFF_RING % 128 == 0 && STAGE_BYTES % 128 == 0 && ST_B % 128 == 0 && ST_Y % 16 == 0, "bulk-copy alignment");
static_assert((2 * NS3 + 2 * NG3 + NS3) * 8 <= 128, "barrier block");

// baked structure packed i | j << 8 | k << 16, in constant memory for the start-up comparison with the run-time table
struct PackedTab3 {
    uint32_t v[TAB3::NNZ];
};
constexpr PackedTab3 make_packed_tab3() {
    PackedTab3 t{};
    for (int n = 0; n < TAB3::NNZ; ++n) t.v[n] = (uint32_t)TAB3::I(n) | ((uint32_t)TAB3::J(n) << 8) | ((uint32_t)TAB3::K(n) << 16);
    return t;
}
__constant__ PackedTab3 c_tab3 = make_packed_tab3();

struct EdgeIn {  // what one consumer warp reads from shared memory for one edge
    float2 go2[4];
    float go_r;
    float Yv[3], wv[3];
};

template <int ROLE>
struct Rows3 {
    static constexpr int R0 = ROLE == 0 ? 1 : ROLE == 1 ? 4 : 0;
    static constexpr int R1 = ROLE == 0 ? 2 : ROLE == 1 ? 5 : 7;
    static constexpr int R2 = ROLE == 0 ? 3 : ROLE == 1 ? 6 : 8;
    __host__ __device__ static constexpr int row(int r) { return r == 0 ? R0 : r == 1 ? R1 : R2; }
    __host__ __device__ static constexpr int local(int i) { return i == R0 ? 0 : i == R1 ? 1 : i == R2 ? 2 : -1; }
};

// DBG: build with the stage knock-outs (tools/time_tp3.py); UNR: unroll factor of the edge run
template <bool DBG, int UNR>
__global__ void __launch_bounds__(128, 4) tp_bwd3_kernel(const Params3 p) {
    const int dbg = DBG ? p.debug : 0;
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BARS);
    int2* s_meta = reinterpret_cast<int2*>(smem + OFF_META);
    float* s_gam = reinterpret_cast<float*>(smem + OFF_GAM);
    float* s_xg = reinterpret_cast<float*>(smem + OFF_XG);
    float* s_xw = reinterpret_cast<float*>(smem + OFF_XW);
    float* s_xb = reinterpret_cast<float*>(smem + OFF_XB);
    float* s_ty = reinterpret_cast<float*>(smem + OFF_TY);
    uint8_t* ring = smem + OFF_RING;
    const uint32_t bar0 = smem_u32(bars);
    auto full_bar = [&](int s) { return bar0 + 8u * s; };
    auto empty_bar = [&](int s) { return bar0 + 8u * (NS3 + s); };
    auto gfull_bar = [&](int g) { return bar0 + 8u * (2 * NS3 + g); };
    auto gempty_bar = [&](int g) { return bar0 + 8u * (2 * NS3 + NG3 + g); };
    auto xfull_bar = [&](int s) { return bar0 + 8u * (2 * NS3 + 2 * NG3 + s); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // the run-time table must have the baked structure; otherwise this kernel does nothing and the two-warp kernel
    // (launched right behind with the complementary test) does the work
    {
        int ok = 1;
        for (int n = threadIdx.x; n < TAB3::NNZ; n += blockDim.x)
            if (((uint32_t)p.tab[3 * n] | ((uint32_t)p.tab[3 * n + 1] << 8) | ((uint32_t)p.tab[3 * n + 2] << 16)) != c_tab3.v[n]) ok = 0;
        if (!__syncthreads_and(ok)) return;
    }
    if (threadIdx.x == 0) {
        for (int s = 0; s < NS3; ++s) {
            mbar_init(full_bar(s), 33);  // 1 expect_tx arrive + 32 cp.async (Y rows) arrivals
            mbar_init(empty_bar(s), 3);
            mbar_init(xfull_bar(s), 1);
        }
        for (int g = 0; g < NG3; ++g) {
            mbar_init(gfull_bar(g), 1);
            mbar_init(gempty_bar(g), 3);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // this CTA's contiguous range of centres / edges
    const int64_t G = gridDim.x, b = blockIdx.x;
    const int64_t c_lo = cut_centre(p.row_ptr, p.ctr, p.N, p.E, b, G);
    const int64_t c_hi = cut_centre(p.row_ptr, p.ctr, p.N, p.E, b + 1, G);
    const int64_t e_lo = p.row_ptr[c_lo], e_hi = p.row_ptr[c_hi];
    constexpr uint32_t GAM_BYTES = D3 * U3 * 4;

    if (warp == 3) {
        // =============================== producer ===============================
        int stage = 0, gslot = 0;
        uint32_t phase = 0, gphase = 0;
        int64_t c_iss = c_lo;
        // gamma rows run ahead of the edge stages (same rule as tp_stream.cu: blocking waits only for centres that begin
        // inside already issued stages, look-ahead centres just end the pass when the ring is busy)
        auto issue_gammas = [&](int64_t issued_end, int64_t look_end) {
            while (c_iss < c_hi) {
                const int rb = p.row_ptr[c_iss], re = p.row_ptr[c_iss + 1];
                if (rb >= look_end) break;
                if (re > rb) {
                    if (rb < issued_end) mbar_wait_backoff(gempty_bar(gslot), gphase ^ 1);
                    else if (!mbar_test(gempty_bar(gslot), gphase ^ 1)) break;
                    s_meta[gslot] = make_int2((int)c_iss, re);
                    mbar_expect_tx(gfull_bar(gslot), GAM_BYTES);
                    bulk_g2s(smem_u32(s_gam + gslot * D3 * U3), p.gamma + c_iss * D3 * U3, GAM_BYTES, gfull_bar(gslot));
                    if (++gslot == NG3) { gslot = 0; gphase ^= 1; }
                }
                ++c_iss;
            }
        };
        if (lane == 0) issue_gammas(e_lo, e_lo + TE3);
        for (int64_t za = e_lo; za < e_hi; za += TE3) {
            const int n = (int)((e_hi - za) < TE3 ? (e_hi - za) : TE3);
            if (lane == 0) {
                if (dbg & 8) mbar_wait(empty_bar(stage), phase ^ 1);
                else mbar_wait_backoff(empty_bar(stage), phase ^ 1);
            }
            __syncwarp();
            uint8_t* sb = ring + stage * STAGE_BYTES;
            if (lane == 0) {
                const uint32_t bytesA = (uint32_t)(n * NIR3 * U3 * 4), bytesB = (uint32_t)(n * D3 * U3 * 4);
                if (dbg & 64) {  // compute only: no edge data is copied, the consumers work on whatever the ring holds
                    mbar_arrive(full_bar(stage));
                } else {
                    mbar_expect_tx(full_bar(stage), bytesA + bytesB);
                    bulk_g2s(smem_u32(sb + ST_A), p.w0 + za * (NIR3 * U3), bytesA, full_bar(stage));
                    bulk_g2s(smem_u32(sb + ST_B), p.gVout + za * (D3 * U3), bytesB, full_bar(stage));
                }
            }
            {
                const float* __restrict__ ysrc = p.Y + za * D3;
                const uint32_t ydst = smem_u32(sb + ST_Y);
                if (!(dbg & (16 | 64)))
                    for (int e = lane; e < n * D3; e += 32) {
                        const int r = e / D3, i = e - r * D3;
                        cp_async4(ydst + 4u * (r * YP3 + i), ysrc + e);
                    }
                cp_async_arrive_noinc(full_bar(stage));
            }
            if (lane == 0) issue_gammas(za + n, za + n + TE3);
            if (++stage == NS3) { stage = 0; phase ^= 1; }
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
        return;
    }

    // =============================== consumers ===============================
    auto run = [&](auto role_tag) {
        constexpr int ROLE = decltype(role_tag)::value;
        using RW = Rows3<ROLE>;
        float2 M2[3][4], gM2[3][4];
        float Mr[3], gMr[3];
        int stage = 0, gslot = 0;
        uint32_t phase = 0, gphase = 0;
        int64_t c = -1, c_prev = c_lo - 1;
        int row_end32 = (int)e_lo;
        int parity_c = 0;

        auto zero_ggamma = [&](int64_t ca, int64_t cb) {  // centres without edges in (ca, cb): ggamma = 0
            for (int64_t cc = ca + 1; cc < cb; ++cc)
                for (int j = ROLE; j < D3; j += 3) p.ggamma[(cc * D3 + j) * U3 + lane] = 0.f;
        };
        auto begin_centre = [&]() {
            mbar_wait(gfull_bar(gslot), gphase);
            const int2 mt = s_meta[gslot];
            c = mt.x;
            row_end32 = mt.y;
            zero_ggamma(c_prev, c);
            c_prev = c;
            const float* __restrict__ gam = s_gam + gslot * D3 * U3 + lane;
            float g[D3];
#pragma unroll
            for (int j = 0; j < D3; ++j) g[j] = gam[j * U3];
            __syncwarp();
            if (lane == 0) mbar_arrive(gempty_bar(gslot));
            if (++gslot == NG3) { gslot = 0; gphase ^= 1; }
#pragma unroll
            for (int r = 0; r < 3; ++r) {
#pragma unroll
                for (int kp = 0; kp < 4; ++kp) {
                    M2[r][kp] = make_float2(0.f, 0.f);
                    gM2[r][kp] = make_float2(0.f, 0.f);
                }
                Mr[r] = 0.f;
                gMr[r] = 0.f;
            }
            if (dbg & 32) return;
#pragma unroll
            for (int n = 0; n < TAB3::NNZ; ++n) {
                const int ti = TAB3::I(n), tj = TAB3::J(n), tk = TAB3::K(n);
                const int r = RW::local(ti);
                if (r >= 0) {
                    const float v = __ldg(p.cgw + n * U3 + lane) * g[tj];
                    if (tk == 8) Mr[r] += v;
                    else if (tk & 1) M2[r][tk >> 1].y += v;
                    else M2[r][tk >> 1].x += v;
                }
            }
        };
        auto end_centre = [&]() {
            // partial ggamma[j] over the table entries whose row belongs to this warp; B and C hand theirs to A
            float gg[D3];
#pragma unroll
            for (int j = 0; j < D3; ++j) gg[j] = 0.f;
#pragma unroll
            for (int n = 0; n < TAB3::NNZ; ++n) {
                const int ti = TAB3::I(n), tj = TAB3::J(n), tk = TAB3::K(n);
                const int r = RW::local(ti);
                if (r >= 0) {
                    const float gm = tk == 8 ? gMr[r] : (tk & 1) ? gM2[r][tk >> 1].y : gM2[r][tk >> 1].x;
                    gg[tj] = fmaf(__ldg(p.cgw + n * U3 + lane), gm, gg[tj]);
                }
            }
            float* xg = s_xg + parity_c * (2 * D3 * U3);
            if (ROLE != 0) {
#pragma unroll
                for (int j = 0; j < D3; ++j) xg[((ROLE - 1) * D3 + j) * U3 + lane] = gg[j];
            }
            named_bar(1, 96);
            if (ROLE == 0) {
#pragma unroll
                for (int j = 0; j < D3; ++j) p.ggamma[(c * D3 + j) * U3 + lane] = (gg[j] + xg[j * U3 + lane]) + xg[(D3 + j) * U3 + lane];
            }
            parity_c ^= 1;
        };

        float* __restrict__ gw0_p = p.gw0 + e_lo * (NIR3 * U3) + lane;
        const int e_lo32 = (int)e_lo, e_hi32 = (int)e_hi;
        for (int za = e_lo32; za < e_hi32; za += TE3) {
            const int n = (e_hi32 - za) < TE3 ? (e_hi32 - za) : TE3;
            mbar_wait(full_bar(stage), phase);
            const uint8_t* sb = ring + stage * STAGE_BYTES;
            const float* __restrict__ sA = reinterpret_cast<const float*>(sb + ST_A) + lane;
            const float* __restrict__ sY = reinterpret_cast<const float*>(sb + ST_Y);
            const float* __restrict__ sB = reinterpret_cast<const float*>(sb + ST_B) + lane;
            [[maybe_unused]] float* __restrict__ xw = s_xw + stage * (TE3 * U3) + lane;
            [[maybe_unused]] float* __restrict__ xb = s_xb + lane;
            float* __restrict__ ty = s_ty + ROLE * (TE3 * 3 * 16) + (lane & 15);
            auto load_edge = [&](int te, EdgeIn& e) {
#pragma unroll
                for (int kp = 0; kp < 4; ++kp) e.go2[kp] = make_float2(sB[(te * D3 + 2 * kp) * U3], sB[(te * D3 + 2 * kp + 1) * U3]);
                e.go_r = sB[(te * D3 + 8) * U3];
                if constexpr (ROLE == 0) {
                    const float4 y4 = *reinterpret_cast<const float4*>(sY + te * YP3);
                    e.Yv[0] = y4.y; e.Yv[1] = y4.z; e.Yv[2] = y4.w;
                    const float w1 = sA[(te * NIR3 + 1) * U3];
                    e.wv[0] = w1; e.wv[1] = w1; e.wv[2] = w1;
                } else if constexpr (ROLE == 1) {
                    const float4 y4 = *reinterpret_cast<const float4*>(sY + te * YP3 + 4);
                    e.Yv[0] = y4.x; e.Yv[1] = y4.y; e.Yv[2] = y4.z;
                    const float w2 = sA[(te * NIR3 + 2) * U3];
                    e.wv[0] = w2; e.wv[1] = w2; e.wv[2] = w2;
                } else {
                    e.Yv[0] = sY[te * YP3];
                    e.Yv[1] = sY[te * YP3 + 7];
                    e.Yv[2] = sY[te * YP3 + 8];
                    e.wv[0] = sA[(te * NIR3) * U3];
                    const float w2 = sA[(te * NIR3 + 2) * U3];
                    e.wv[1] = w2; e.wv[2] = w2;
                }
            };
            int t = 0;
            while (t < n) {
                if (za + t == row_end32) {  // warp-uniform: first edge of the next non-empty centre
                    if (c >= 0 && !(dbg & 32)) end_centre();
                    begin_centre();
                }
                const int t_end = (row_end32 - za) < n ? (row_end32 - za) : n;
                if (dbg & 1) t = t_end;
                // (a hand-made software pipeline -- reads of edge t + 1 issued before the arithmetic of edge t -- costs
                // more registers and moves than it hides)
#pragma unroll UNR
                for (; t < t_end; ++t) {
                    EdgeIn cur;
                    load_edge(t, cur);
                    float gin[3], v[3];
#pragma unroll
                    for (int r = 0; r < 3; ++r) {
                        v[r] = cur.Yv[r] * cur.wv[r];
                        const float2 vv = make_float2(v[r], v[r]);
                        float2 a2 = make_float2(0.f, 0.f);
#pragma unroll
                        for (int kp = 0; kp < 4; ++kp) {
                            a2 = fma2(M2[r][kp], cur.go2[kp], a2);
                            gM2[r][kp] = fma2(vv, cur.go2[kp], gM2[r][kp]);
                        }
                        gin[r] = fmaf(Mr[r], cur.go_r, a2.x + a2.y);
                        gMr[r] = fmaf(v[r], cur.go_r, gMr[r]);
                    }
                    // Vin[i] = Y[i] w0[l(i)]:  gw0[l] = sum_{i in l} Y[i] gin[i]
                    if constexpr (ROLE == 0) {
                        gw0_p[1 * U3] = fmaf(cur.Yv[2], gin[2], fmaf(cur.Yv[1], gin[1], cur.Yv[0] * gin[0]));
                    } else if constexpr (ROLE == 1) {
                        xb[t * U3] = fmaf(cur.Yv[2], gin[2], fmaf(cur.Yv[1], gin[1], cur.Yv[0] * gin[0]));
                    } else {
                        gw0_p[0] = cur.Yv[0] * gin[0];
                        xw[t * U3] = fmaf(cur.Yv[2], gin[2], cur.Yv[1] * gin[1]);
                    }
                    // gY[z][i] += sum_u w0[l(i)][u] gin[i][u]: one xor-16 step in registers (three independent shuffles, no
                    // chain), lanes 0-15 park the half sums; the stage's rows are summed once per stage below, instead of
                    // a five-level shuffle chain per edge on the edge's critical path.
                    if (!(dbg & 2)) {
#pragma unroll
                        for (int r = 0; r < 3; ++r) {
                            float pr = cur.wv[r] * gin[r];
                            pr += __shfl_xor_sync(0xffffffffu, pr, 16);
                            if (lane < 16) ty[(t * 3 + r) * 16] = pr;
                        }
                    }
                    gw0_p += NIR3 * U3;
                }
            }
            __syncwarp();
            if (!(dbg & 2) && lane < 3 * n) {
                // lane j sums row j = (edge j / 3, local row j % 3) of the tile: 16 floats, chunk order rotated per lane
                // so that the eight lanes of a 128-bit phase hit eight different bank groups
                const float4* __restrict__ row = reinterpret_cast<const float4*>(ty - (lane & 15) + lane * 16);
                const int sw = (lane >> 1) & 3;
                const float4 a = row[sw], b4 = row[1 ^ sw], c4 = row[2 ^ sw], d4 = row[3 ^ sw];
                const float tot = (((a.x + a.y) + (a.z + a.w)) + ((b4.x + b4.y) + (b4.z + b4.w))) + (((c4.x + c4.y) + (c4.z + c4.w)) + ((d4.x + d4.y) + (d4.z + d4.w)));
                const int tt = lane / 3, r = lane - 3 * tt;
                if (!(dbg & 4)) atomicAdd(p.gY + (int64_t)(za + tt) * D3 + (r == 0 ? RW::R0 : r == 1 ? RW::R1 : RW::R2), tot);  // RED, one writer per address
            }
            __syncwarp();
            if constexpr (ROLE == 2) {
                if (lane == 0) mbar_arrive(xfull_bar(stage));  // C's l = 2 partials of this stage are in the slot
            }
            if constexpr (ROLE == 1) {
                mbar_wait(xfull_bar(stage), phase);
                float* __restrict__ o = p.gw0 + (int64_t)za * (NIR3 * U3) + 2 * U3 + lane;
#pragma unroll 4
                for (int tt = 0; tt < n; ++tt) o[tt * (NIR3 * U3)] = xb[tt * U3] + xw[tt * U3];
                __syncwarp();
            }
            if (lane == 0) mbar_arrive(empty_bar(stage));
            if (++stage == NS3) { stage = 0; phase ^= 1; }
        }
        if (c >= 0) end_centre();
        zero_ggamma(c_prev, c_hi);
    };
    if (warp == 0) run(std::integral_constant<int, 0>{});
    else if (warp == 1) run(std::integral_constant<int, 1>{});
    else run(std::integral_constant<int, 2>{});
}

}  // namespace

// returns 0 if launched (the kernel itself stands down when the table does not have the baked structure: the caller
// launches the two-warp kernel with skip_if_baked right behind), -1 if not eligible
int ab2_tp_stream3_bwd(int64_t N, int64_t E, const int32_t* tab, const void* cgw, const int32_t* row_ptr, const int32_t* ctr, const void* gamma,
                       const void* Y, const void* w0, const void* gVout, void* gw0, void* gY, void* ggamma, cudaStream_t st) {
    if (!g_ab2_opt_tp_stream3 || E <= 0 || N <= 0 || E >= ((int64_t)1 << 31)) return -1;
    static int num_sms = 0, cps = 0;
    using KernT = void (*)(const Params3);
    static const KernT kerns[4] = {tp_bwd3_kernel<false, 2>, tp_bwd3_kernel<false, 1>, tp_bwd3_kernel<true, 2>, tp_bwd3_kernel<true, 1>};
    if (num_sms == 0) {
        int dev = 0, max_smem = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        cps = 1 << 30;
        for (KernT k : kerns) {
            int c1 = 0;
            if (SMEM3 > max_smem || cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM3) != cudaSuccess ||
                cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c1, k, 128, SMEM3) != cudaSuccess || c1 < 1) {
                cudaGetLastError();
                c1 = -1;
            }
            if (c1 < cps) cps = c1;
        }
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
    }
    if (cps < 1) return -1;
    extern int g_ab2_opt_tp_stream_cps;
    const int use = (g_ab2_opt_tp_stream_cps > 0 && g_ab2_opt_tp_stream_cps < cps) ? g_ab2_opt_tp_stream_cps : cps;
    int64_t grid = (int64_t)num_sms * use;
    if (grid > N) grid = N;
    Params3 p;
    p.N = N; p.E = E; p.tab = tab; p.cgw = (const float*)cgw; p.row_ptr = row_ptr; p.ctr = ctr; p.gamma = (const float*)gamma;
    p.Y = (const float*)Y; p.w0 = (const float*)w0; p.gVout = (const float*)gVout; p.gw0 = (float*)gw0; p.gY = (float*)gY; p.ggamma = (float*)ggamma;
    p.debug = g_ab2_opt_tp_stream3_debug & 0xff;
    const int unr1 = ((g_ab2_opt_tp_stream3_debug >> 8) & 1) ^ 1;  // default: the unroll-1 build; bit 8 selects unroll 2
    kerns[(p.debug ? 2 : 0) + unr1]<<<(unsigned)grid, 128, SMEM3, st>>>(p);
    return 0;
}

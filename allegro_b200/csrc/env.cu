// Per-centre environment sum and its adjoint.
//
// Reference: MakeWeightedChannels (allegro/nn/_strided/_channels.py:44-57) builds
// A[z][u][j] = Y[z][j] * w[z][u][irrep(j)] for every edge, Contracter.forward
// (_contract.py:195-205) scales by 1/sqrt(avg_num_neighbors), scatter-sums over the centre and
// gathers the sum back per edge.  With centre-sorted edges the sum is a reduction over a
// contiguous row; A is never materialised and the gather is a broadcast read of gamma[c].
//
// Layouts: Y[E][D] (TAcc), w[z][n_ir][U] (TAct, leading dim w_ld), gamma[N][D][U] (TAcc).
#include "common.cuh"

extern int g_ab2_opt_env_split;
int g_ab2_opt_env_unroll = 2;  // edge-loop unroll of env_sum with 4 warps per centre: 2 or 4  // warps per (centre, channel chunk) in env_sum / env_bwd: 1, 2 or 4

// SPLIT warps of one CTA share a (centre, 32-channel chunk): each streams every SPLIT-th edge of the
// row, the partial sums meet in shared memory.  One warp per centre (SPLIT = 1) leaves only ~2 waves
// of long serial loops (42 edges/centre on c2) and is latency-bound at ~50 % of the HBM rate.
template <typename TAct, typename TAcc, int LMAX, int SPLIT, int UNR = 2>
__global__ void __launch_bounds__(128) env_sum_kernel(int64_t N, int U, const int32_t* __restrict__ row_ptr,
                                                      const TAcc* __restrict__ Y, const TAct* __restrict__ w, int64_t w_ld,
                                                      TAcc sf, TAcc* __restrict__ gamma) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    __shared__ TAcc red[SPLIT > 1 ? 4 : 1][SPLIT > 1 ? D : 1][32];
    const int nchunk = (U + 31) >> 5;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t grp = ((int64_t)blockIdx.x * 4 + warp) / SPLIT;
    const int sub = warp % SPLIT;
    const int64_t c = grp / nchunk;
    const bool valid = c < N;
    const int u = (int)(grp % nchunk) * 32 + lane;
    const bool live = valid && u < U;
    const int beg = valid ? row_ptr[c] : 0, end = valid ? row_ptr[c + 1] : 0;
    TAcc acc[D];
#pragma unroll
    for (int j = 0; j < D; ++j) acc[j] = TAcc(0);
#pragma unroll UNR
    for (int z = beg + sub; z < end; z += SPLIT) {
        const TAcc* __restrict__ Yz = Y + (int64_t)z * D;
        const TAct* __restrict__ wz = w + (int64_t)z * w_ld;
#pragma unroll
        for (int l = 0; l <= LMAX; ++l) {
            const TAcc wl = live ? to_acc<TAcc>(wz[l * U + u]) : TAcc(0);
#pragma unroll
            for (int j = l * l; j < (l + 1) * (l + 1); ++j) acc[j] += Yz[j] * wl;
        }
    }
    if constexpr (SPLIT > 1) {
        if (sub != 0) {
#pragma unroll
            for (int j = 0; j < D; ++j) red[warp][j][lane] = acc[j];
        }
        __syncthreads();
        if (sub == 0) {
#pragma unroll
            for (int t = 1; t < SPLIT; ++t) {
#pragma unroll
                for (int j = 0; j < D; ++j) acc[j] += red[warp + t][j][lane];
            }
        }
    }
    if (live && sub == 0) {
#pragma unroll
        for (int j = 0; j < D; ++j) gamma[((int64_t)c * D + j) * U + u] = sf * acc[j];
    }
}

// One warp per edge.  gw[z][l][u] = sf * sum_{j in l} Y[z][j] ggamma[c][j][u];
// gY[z][j] += sf * sum_u w[z][l(j)][u] ggamma[c][j][u]  (warp-shuffle reduction over u).
template <typename TAct, typename TAcc, int LMAX>
__global__ void __launch_bounds__(128) env_bwd_kernel(int64_t E, int U, const int32_t* __restrict__ ctr, const TAcc* __restrict__ Y,
                                                      const TAct* __restrict__ w, int64_t w_ld, const TAcc* __restrict__ ggamma,
                                                      TAcc sf, TAct* __restrict__ gw, int64_t gw_ld, TAcc* __restrict__ gY) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    const int64_t z = ((int64_t)blockIdx.x * 128 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (z >= E) return;
    const int64_t c = ctr[z];
    TAcc Yz[D], gy[D];
#pragma unroll
    for (int j = 0; j < D; ++j) {
        Yz[j] = Y[z * D + j];
        gy[j] = TAcc(0);
    }
    for (int u = lane; u < U; u += 32) {
#pragma unroll
        for (int l = 0; l <= LMAX; ++l) {
            const TAcc wl = to_acc<TAcc>(w[z * w_ld + l * U + u]);
            TAcc gwl = TAcc(0);
#pragma unroll
            for (int j = l * l; j < (l + 1) * (l + 1); ++j) {
                const TAcc ga = sf * ggamma[(c * D + j) * U + u];
                gwl += Yz[j] * ga;
                gy[j] += wl * ga;
            }
            gw[z * gw_ld + l * U + u] = from_acc<TAct>(gwl);
        }
    }
#pragma unroll
    for (int j = 0; j < D; ++j) {
        const TAcc s = warp_sum(gy[j]);
        if (lane == (j & 31)) gY[z * D + j] += s;
    }
}

// Warp per (centre, 32-channel chunk): ggamma[c][.][u] is loaded once into registers and the
// centre's edges are streamed (two in flight).  Same arithmetic as env_bwd_kernel.
template <typename TAct, typename TAcc, int LMAX, int SPLIT>
__global__ void __launch_bounds__(128) env_bwd_fast_kernel(int64_t N, int U, const int32_t* __restrict__ row_ptr,
                                                           const TAcc* __restrict__ Y, const TAct* __restrict__ w, int64_t w_ld,
                                                           const TAcc* __restrict__ ggamma, TAcc sf, TAct* __restrict__ gw,
                                                           int64_t gw_ld, TAcc* __restrict__ gY) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    const int nchunk = (U + 31) >> 5;
    const int64_t wid = ((int64_t)blockIdx.x * 128 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int64_t grp = wid / SPLIT;  // SPLIT warps stream interleaved edges of one (centre, chunk)
    const int sub = (int)(wid % SPLIT);
    const int64_t c = grp / nchunk;
    if (c >= N) return;
    const int u = (int)(grp % nchunk) * 32 + lane;
    const bool live = u < U;
    const int beg = row_ptr[c], end = row_ptr[c + 1];
    TAcc gg[D];
#pragma unroll
    for (int j = 0; j < D; ++j) gg[j] = live ? sf * ggamma[(c * D + j) * U + u] : TAcc(0);
#pragma unroll 2
    for (int64_t z = beg + sub; z < end; z += SPLIT) {
        TAcc Yz[D], wl[LMAX + 1];
#pragma unroll
        for (int j = 0; j < D; ++j) Yz[j] = Y[z * D + j];
#pragma unroll
        for (int l = 0; l <= LMAX; ++l) wl[l] = live ? to_acc<TAcc>(w[z * w_ld + l * U + u]) : TAcc(0);
        TAcc part[D];
#pragma unroll
        for (int l = 0; l <= LMAX; ++l) {
            TAcc gwl = TAcc(0);
#pragma unroll
            for (int j = l * l; j < (l + 1) * (l + 1); ++j) {
                gwl += Yz[j] * gg[j];
                part[j] = wl[l] * gg[j];
            }
            if (live) gw[z * gw_ld + l * U + u] = from_acc<TAct>(gwl);
        }
        const TAcc tot = warp_multi_sum<TAcc, D>(part, lane);
        const int j = lane >> 1;
        if (!(lane & 1) && j < D) {
            if (nchunk == 1) gY[z * D + j] += tot;
            else atomicAdd(&gY[z * D + j], tot);
        }
    }
}

extern "C" int ab2_env_sum(int dtype, int lmax, int64_t N, int U, const int32_t* row_ptr, const void* Y, const void* w,
                           int64_t w_ld, double sf, void* gamma, void* stream) {
    if (N == 0) return 0;
    AB2_CHECK_ARG(row_ptr && Y && w && gamma && U > 0, "null pointer / U");
    AB2_CHECK_ARG(w_ld >= (int64_t)(lmax + 1) * U, "w_ld too small");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t groups = N * ((U + 31) / 32);
    // auto (0): 4 warps per centre when one warp would cover all channels (U <= 32: +85 % on c2),
    // one otherwise (U = 64 measured slower when split)
    const int split = g_ab2_opt_env_split ? g_ab2_opt_env_split : (U <= 32 ? 4 : 1);
    if (split >= 4 && g_ab2_opt_env_unroll == 4) {
        AB2_DISPATCH_DTYPE(dtype, AB2_DISPATCH_LMAX(lmax, env_sum_kernel<TAct, TAcc, LMAX, 4, 4><<<ab2_blocks(groups * 4 * 32, 128), 128, 0, st>>>(
                                                              N, U, row_ptr, (const TAcc*)Y, (const TAct*)w, w_ld, (TAcc)sf, (TAcc*)gamma)));
    } else if (split >= 4) {
        AB2_DISPATCH_DTYPE(dtype, AB2_DISPATCH_LMAX(lmax, env_sum_kernel<TAct, TAcc, LMAX, 4><<<ab2_blocks(groups * 4 * 32, 128), 128, 0, st>>>(
                                                              N, U, row_ptr, (const TAcc*)Y, (const TAct*)w, w_ld, (TAcc)sf, (TAcc*)gamma)));
    } else if (split >= 2) {
        AB2_DISPATCH_DTYPE(dtype, AB2_DISPATCH_LMAX(lmax, env_sum_kernel<TAct, TAcc, LMAX, 2><<<ab2_blocks(groups * 2 * 32, 128), 128, 0, st>>>(
                                                              N, U, row_ptr, (const TAcc*)Y, (const TAct*)w, w_ld, (TAcc)sf, (TAcc*)gamma)));
    } else {
        AB2_DISPATCH_DTYPE(dtype, AB2_DISPATCH_LMAX(lmax, env_sum_kernel<TAct, TAcc, LMAX, 1><<<ab2_blocks(groups * 32, 128), 128, 0, st>>>(
                                                              N, U, row_ptr, (const TAcc*)Y, (const TAct*)w, w_ld, (TAcc)sf, (TAcc*)gamma)));
    }
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern int g_ab2_opt_tp_fast;
int ab2_env_bwd_stream(int dtype, int lmax, int64_t N, int64_t E, int U, const int32_t* ctr, const void* Y, const void* w, int64_t w_ld,
                       const void* ggamma, double sf, void* gw, int64_t gw_ld, void* gY, cudaStream_t st);

extern "C" int ab2_env_bwd(int dtype, int lmax, int64_t N, int64_t E, int U, const int32_t* row_ptr, const int32_t* ctr, const void* Y,
                           const void* w, int64_t w_ld, const void* ggamma, double sf, void* gw, int64_t gw_ld, void* gY,
                           void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(ctr && Y && w && ggamma && gw && gY && U > 0, "null pointer / U");
    cudaStream_t st = (cudaStream_t)stream;
    if (g_ab2_opt_tp_fast && ab2_env_bwd_stream(dtype, lmax, N, E, U, ctr, Y, w, w_ld, ggamma, sf, gw, gw_ld, gY, st) == 0) {
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    }
    if (g_ab2_opt_tp_fast && row_ptr && lmax <= 3) {
        // auto (0): split only when a centre needs several channel chunks (U > 32)
        const int opt = g_ab2_opt_env_split ? g_ab2_opt_env_split : (U > 32 && dtype != AB2_F64 ? 4 : 1);
        const int split = opt >= 4 ? 4 : opt >= 2 ? 2 : 1;
        const int64_t warps = N * ((U + 31) / 32) * split;
#define AB2_ENV_BWD(L, SP)                                                                                              \
    AB2_DISPATCH_DTYPE(dtype, env_bwd_fast_kernel<TAct, TAcc, L, SP><<<ab2_blocks(warps * 32, 128), 128, 0, st>>>(           \
                                  N, U, row_ptr, (const TAcc*)Y, (const TAct*)w, w_ld, (const TAcc*)ggamma, (TAcc)sf, (TAct*)gw, gw_ld, (TAcc*)gY))
#define AB2_ENV_BWD_L(L)                                  \
    do {                                                  \
        if (split == 4) { AB2_ENV_BWD(L, 4); }            \
        else if (split == 2) { AB2_ENV_BWD(L, 2); }       \
        else { AB2_ENV_BWD(L, 1); }                       \
    } while (0)
        if (lmax == 3) AB2_ENV_BWD_L(3);
        else if (lmax == 2) AB2_ENV_BWD_L(2);
        else if (lmax == 1) AB2_ENV_BWD_L(1);
        else AB2_ENV_BWD_L(0);
#undef AB2_ENV_BWD_L
#undef AB2_ENV_BWD
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    }
    AB2_DISPATCH_DTYPE(dtype, AB2_DISPATCH_LMAX(lmax, env_bwd_kernel<TAct, TAcc, LMAX><<<ab2_blocks(E * 32, 128), 128, 0, st>>>(
                                                          E, U, ctr, (const TAcc*)Y, (const TAct*)w, w_ld, (const TAcc*)ggamma, (TAcc)sf,
                                                          (TAct*)gw, gw_ld, (TAcc*)gY)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

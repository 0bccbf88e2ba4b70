// Error plumbing, spherical-harmonic edge embedding (fwd/bwd), edge->atom energy reduction,
// force assembly and layout helpers.
#include <cstdarg>

#include "common.cuh"
#include "sh_generated.cuh"

static thread_local char g_err[1024] = "";

void ab2_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int g_ab2_opt_tp_fast = 1;
int g_ab2_opt_linear_tc = 1;
int g_ab2_opt_linear_tma = 1;  // TMA-producer variant of the tensor-core linear where eligible
int g_ab2_opt_tc_debug = 0;
int g_ab2_opt_env_split = 0;  // 0: auto (env.cu)
extern int g_ab2_opt_tp_variant;
extern int g_ab2_opt_tp_stream, g_ab2_opt_tp_stream_te, g_ab2_opt_tp_stream_cps;
extern int g_ab2_opt_env_stream, g_ab2_opt_env_stream_cps, g_ab2_opt_env_unroll;
extern int g_ab2_opt_tp_stream3, g_ab2_opt_tp_stream3_debug, g_ab2_opt_tp_stream_gytile, g_ab2_opt_tp_stream_last, g_ab2_opt_tp_baked64;

extern "C" const char* ab2_last_error(void) { return g_err; }
extern "C" int ab2_set_option(const char* key, int value) {
    if (!key) return 1;
    if (!strcmp(key, "tp_fast")) { g_ab2_opt_tp_fast = value; return 0; }
    if (!strcmp(key, "linear_tc")) { g_ab2_opt_linear_tc = value; return 0; }
    if (!strcmp(key, "linear_tma")) { g_ab2_opt_linear_tma = value; return 0; }
    if (!strcmp(key, "tc_debug")) { g_ab2_opt_tc_debug = value; return 0; }
    if (!strcmp(key, "env_split")) { g_ab2_opt_env_split = value; return 0; }
    if (!strcmp(key, "tp_variant")) { g_ab2_opt_tp_variant = value; return 0; }
    if (!strcmp(key, "env_stream_cps")) { g_ab2_opt_env_stream_cps = value; return 0; }
    if (!strcmp(key, "env_unroll")) { g_ab2_opt_env_unroll = value; return 0; }
    if (!strcmp(key, "env_stream")) { g_ab2_opt_env_stream = value; return 0; }
    if (!strcmp(key, "tp_stream")) { g_ab2_opt_tp_stream = value; return 0; }
    if (!strcmp(key, "tp_baked64")) { g_ab2_opt_tp_baked64 = value; return 0; }
    if (!strcmp(key, "tp_stream_last")) { g_ab2_opt_tp_stream_last = value; return 0; }
    if (!strcmp(key, "tp_stream_gytile")) { g_ab2_opt_tp_stream_gytile = value; return 0; }
    if (!strcmp(key, "tp_stream3")) { g_ab2_opt_tp_stream3 = value; return 0; }
    if (!strcmp(key, "tp_stream3_debug")) { g_ab2_opt_tp_stream3_debug = value; return 0; }
    if (!strcmp(key, "tp_stream_te")) { g_ab2_opt_tp_stream_te = value; return 0; }
    if (!strcmp(key, "tp_stream_cps")) { g_ab2_opt_tp_stream_cps = value; return 0; }
    ab2_set_error("unknown option %s", key);
    return 1;
}
extern "C" int ab2_version(void) { return 100; }
extern "C" int ab2_device_ok(void) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return 0; }
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) { cudaGetLastError(); return 0; }
    return (p.major == 9 && p.minor == 0) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------
// Spherical harmonics.  One thread per edge; Y staged through shared memory so the [E][d]
// store is coalesced.
// ---------------------------------------------------------------------------------------
template <typename TAcc, int LMAX>
__global__ void __launch_bounds__(128) sh_fwd_kernel(int64_t E, const TAcc* __restrict__ vec, TAcc* __restrict__ Y) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    __shared__ TAcc sY[128 * D];
    const int64_t z0 = (int64_t)blockIdx.x * 128;
    const int64_t z = z0 + threadIdx.x;
    if (z < E) {
        TAcc x = vec[z * 3 + 0], y = vec[z * 3 + 1], w = vec[z * 3 + 2];
        TAcc inv = TAcc(1) / sqrt(x * x + y * y + w * w);
        TAcc loc[D];
        sh_eval<LMAX, TAcc>(x * inv, y * inv, w * inv, loc);
#pragma unroll
        for (int j = 0; j < D; ++j) sY[threadIdx.x * D + j] = loc[j];
    }
    __syncthreads();
    const int64_t n = min((int64_t)128, E - z0) * D;
    for (int64_t e = threadIdx.x; e < n; e += 128) Y[z0 * D + e] = sY[e];
}

template <typename TAcc, int LMAX>
__global__ void __launch_bounds__(128) sh_bwd_kernel(int64_t E, const TAcc* __restrict__ vec, const TAcc* __restrict__ gY,
                                                     TAcc* __restrict__ gvec, int accumulate) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    __shared__ TAcc sG[128 * D];
    const int64_t z0 = (int64_t)blockIdx.x * 128;
    const int64_t n = min((int64_t)128, E - z0) * D;
    for (int64_t e = threadIdx.x; e < n; e += 128) sG[e] = gY[z0 * D + e];
    __syncthreads();
    const int64_t z = z0 + threadIdx.x;
    if (z >= E) return;
    TAcc x = vec[z * 3 + 0], y = vec[z * 3 + 1], w = vec[z * 3 + 2];
    TAcc inv = TAcc(1) / sqrt(x * x + y * y + w * w);
    x *= inv; y *= inv; w *= inv;
    TAcc g[D];
#pragma unroll
    for (int j = 0; j < D; ++j) g[j] = sG[threadIdx.x * D + j];
    TAcc gx, gy, gz;
    sh_grad<LMAX, TAcc>(x, y, w, g, gx, gy, gz);
    // chain through r_hat = r/|r|:  g_r = (I - r_hat r_hat^T) g / |r|
    TAcc dot = gx * x + gy * y + gz * w;
    gx = (gx - dot * x) * inv;
    gy = (gy - dot * y) * inv;
    gz = (gz - dot * w) * inv;
    if (accumulate) {
        gvec[z * 3 + 0] += gx; gvec[z * 3 + 1] += gy; gvec[z * 3 + 2] += gz;
    } else {
        gvec[z * 3 + 0] = gx; gvec[z * 3 + 1] = gy; gvec[z * 3 + 2] = gz;
    }
}

extern "C" int ab2_sh_fwd(int acc_dtype, int lmax, int64_t E, const void* vec, void* Y, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(vec && Y, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, AB2_DISPATCH_LMAX(lmax, sh_fwd_kernel<TAcc, LMAX><<<ab2_blocks(E, 128), 128, 0, st>>>(
                                                            E, (const TAcc*)vec, (TAcc*)Y)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_sh_bwd(int acc_dtype, int lmax, int64_t E, const void* vec, const void* gY, void* gvec, int accumulate,
                          void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(vec && gY && gvec, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, AB2_DISPATCH_LMAX(lmax, sh_bwd_kernel<TAcc, LMAX><<<ab2_blocks(E, 128), 128, 0, st>>>(
                                                            E, (const TAcc*)vec, (const TAcc*)gY, (TAcc*)gvec, accumulate)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------
// Edge -> atom energy reduction over CSR rows: one warp per centre, shuffle reduction,
// fixed summation order (deterministic).
// ---------------------------------------------------------------------------------------
template <typename TAcc>
__global__ void __launch_bounds__(256) edge_sum_kernel(int64_t N, const int32_t* __restrict__ row_ptr, const TAcc* __restrict__ Ez,
                                                       TAcc factor, TAcc* __restrict__ Ei) {
    const int64_t c = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (c >= N) return;
    const int beg = row_ptr[c], end = row_ptr[c + 1];
    TAcc s = 0;
    for (int z = beg + lane; z < end; z += 32) s += factor * Ez[z];
    s = warp_sum(s);
    if (lane == 0) Ei[c] = s;
}

template <typename TAcc>
__global__ void __launch_bounds__(256) edge_sum_bwd_kernel(int64_t E, const int32_t* __restrict__ ctr, const TAcc* __restrict__ gEi,
                                                           TAcc factor, TAcc* __restrict__ gEz) {
    const int64_t z = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (z < E) gEz[z] = factor * gEi[ctr[z]];
}

extern "C" int ab2_edge_sum(int acc_dtype, int64_t N, const int32_t* row_ptr, const void* Ez, double factor, void* Ei,
                            void* stream) {
    if (N == 0) return 0;
    AB2_CHECK_ARG(row_ptr && Ei, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, edge_sum_kernel<TAcc><<<ab2_blocks(N * 32, 256), 256, 0, st>>>(N, row_ptr, (const TAcc*)Ez,
                                                                                                 (TAcc)factor, (TAcc*)Ei));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_edge_sum_bwd(int acc_dtype, int64_t E, const int32_t* ctr, const void* gEi, double factor, void* gEz,
                                void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(ctr && gEi && gEz, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, edge_sum_bwd_kernel<TAcc><<<ab2_blocks(E, 256), 256, 0, st>>>(E, ctr, (const TAcc*)gEi,
                                                                                                (TAcc)factor, (TAcc*)gEz));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------
// Force assembly.  gvec[z] = dE/d r_z with r_z = pos[nbr] - pos[ctr]:
//   dE/dpos[ctr] -= gvec,  dE/dpos[nbr] += gvec;   F = -dE/dpos
// so F[a] = sum_{z in row a} gvec[z] - sum_{z : nbr[z] = a} gvec[z].  Both sums are SEGMENTED
// reductions: the first over the centre-sorted CSR row, the second over the transposed CSR
// (edges grouped by neighbour: col_ptr[n_total+1], col_perm[E] = edge ids sorted by neighbour,
// built once per neighbour list).  One warp per atom, fixed summation order, no atomics: forces
// are bitwise reproducible from run to run, and F needs no zero-fill.
//
// WITH_W: the same walk also forms the centroid per-atom virial
//   W[a][p][q] = - sum_{z : nbr[z] = a} vec[z][p] gvec[z][q]
// from the column loop (vec gathered through col_perm like gvec).  F's arithmetic is untouched
// by it, so F is bitwise that of the instantiation without W.  The 9 lane sums are reduced in
// the fixed order p-major, q-minor.
// ---------------------------------------------------------------------------------------
template <typename TAcc, bool WITH_W>
__global__ void __launch_bounds__(256) force_scatter_kernel(int64_t N, int64_t n_total, const int32_t* __restrict__ row_ptr,
                                                            const int32_t* __restrict__ col_ptr,
                                                            const int32_t* __restrict__ col_perm, const TAcc* __restrict__ vec,
                                                            const TAcc* __restrict__ gvec, TAcc* __restrict__ F, TAcc* __restrict__ W) {
    const int64_t a = ((int64_t)blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (a >= n_total) return;
    TAcc sx = 0, sy = 0, sz = 0;
    if (a < N) {
        const int beg = row_ptr[a], end = row_ptr[a + 1];
        for (int z = beg + lane; z < end; z += 32) {
            sx += gvec[(int64_t)z * 3 + 0];
            sy += gvec[(int64_t)z * 3 + 1];
            sz += gvec[(int64_t)z * 3 + 2];
        }
    }
    TAcc w[WITH_W ? 9 : 1];
    if (WITH_W) {
#pragma unroll
        for (int k = 0; k < 9; ++k) w[k] = 0;
    }
    const int cb = col_ptr[a], ce = col_ptr[a + 1];
    for (int t = cb + lane; t < ce; t += 32) {
        const int64_t z = col_perm[t];
        const TAcc gx = gvec[z * 3 + 0], gy = gvec[z * 3 + 1], gz = gvec[z * 3 + 2];
        sx -= gx;
        sy -= gy;
        sz -= gz;
        if (WITH_W) {
            const TAcc v[3] = {vec[z * 3 + 0], vec[z * 3 + 1], vec[z * 3 + 2]};
#pragma unroll
            for (int p = 0; p < 3; ++p) {
                w[p * 3 + 0] += v[p] * gx;
                w[p * 3 + 1] += v[p] * gy;
                w[p * 3 + 2] += v[p] * gz;
            }
        }
    }
    sx = warp_sum(sx); sy = warp_sum(sy); sz = warp_sum(sz);
    if (WITH_W) {
#pragma unroll
        for (int k = 0; k < 9; ++k) w[k] = warp_sum(w[k]);
    }
    if (lane == 0) {
        F[a * 3 + 0] = sx;
        F[a * 3 + 1] = sy;
        F[a * 3 + 2] = sz;
        if (WITH_W) {
#pragma unroll
            for (int k = 0; k < 9; ++k) W[a * 9 + k] = -w[k];
        }
    }
}

extern "C" int ab2_force_scatter(int acc_dtype, int64_t N, int64_t n_total, int64_t E, const int32_t* row_ptr,
                                 const int32_t* col_ptr, const int32_t* col_perm, const void* gvec, void* F, void* stream) {
    if (n_total == 0) return 0;
    AB2_CHECK_ARG(row_ptr && col_ptr && gvec && F && (E == 0 || col_perm), "null pointer");
    AB2_CHECK_ARG(N <= n_total, "more centres than atoms");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, force_scatter_kernel<TAcc, false><<<ab2_blocks(n_total * 32, 256), 256, 0, st>>>(
                                    N, n_total, row_ptr, col_ptr, col_perm, nullptr, (const TAcc*)gvec, (TAcc*)F, nullptr));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_force_virial_scatter(int acc_dtype, int64_t N, int64_t n_total, int64_t E, const int32_t* row_ptr,
                                        const int32_t* col_ptr, const int32_t* col_perm, const void* vec, const void* gvec, void* F,
                                        void* W, void* stream) {
    if (n_total == 0) return 0;
    AB2_CHECK_ARG(row_ptr && col_ptr && F && W && (E == 0 || (col_perm && vec && gvec)), "null pointer");
    AB2_CHECK_ARG(N <= n_total, "more centres than atoms");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, force_scatter_kernel<TAcc, true><<<ab2_blocks(n_total * 32, 256), 256, 0, st>>>(
                                    N, n_total, row_ptr, col_ptr, col_perm, (const TAcc*)vec, (const TAcc*)gvec, (TAcc*)F, (TAcc*)W));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------
// [z][u][i] (reference strided layout, _contract.py:209-210)  <->  [z][i][u] (internal)
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) transpose_ui_kernel(int64_t total, int U, int d, const T* __restrict__ src, T* __restrict__ dst,
                                                           int to_internal) {
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= total) return;
    const int64_t z = e / (U * d);
    const int r = (int)(e - z * U * d);
    if (to_internal) {  // dst index e = (z, i, u)
        const int i = r / U, u = r % U;
        dst[e] = src[(z * U + u) * d + i];
    } else {  // dst index e = (z, u, i)
        const int u = r / d, i = r % d;
        dst[e] = src[(z * d + i) * U + u];
    }
}

extern "C" int ab2_transpose_ui(int dtype, int64_t E, int U, int d, const void* src, void* dst, int to_internal, void* stream) {
    const int64_t total = E * U * d;
    if (total == 0) return 0;
    AB2_CHECK_ARG(src && dst, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_DTYPE(dtype, transpose_ui_kernel<TAct><<<ab2_blocks(total, 256), 256, 0, st>>>(total, U, d, (const TAct*)src,
                                                                                                  (TAct*)dst, to_internal));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// Tangent (forward-mode) kernels of the per-edge force path: with the edge vectors moved along vdot, the pipeline's
// multilinear steps (GEMMs, env sums, tensor products, scatters) take their tangents from the existing kernels, one call
// per replaced input; the truly nonlinear steps need the kernels below (DESIGN.md section 4.11):
//   ab2_sh_jvp       Yd = dY/dvec . vdot                                       (spherical harmonics of r/|r|)
//   ab2_sh_hvp       gvec_dot += (d2 sum_k gY_k Y_k / dvec2) . vdot             (the SH adjoint's own curvature)
//   ab2_act_bwd_jvp  gpre_dot = ga_dot phi'(pre) + ga phi''(pre) pre_dot       (the MLP nonlinearity in the adjoint)
//   ab2_zbl_hvp      gvec_dot += (d2 Ez / dvec2) . vdot                         (the ZBL pair term)
// The radial basis' tangents are in radial.cu (they share its Bessel basis), the force-constant gather / fold tangent
// mode in fc.cu.  One thread per edge (per element for the activation), no atomics, so every result is deterministic.
#include "common.cuh"
#include "sh_generated.cuh"
#include "sh_hvp_generated.cuh"

namespace {

// u = r / |r| and the tangent of u along v:  u_dot = (v - (u.v) u) / |r|
template <typename T>
__device__ __forceinline__ void unit_tangent(const T* __restrict__ vec, const T* __restrict__ vdot, int64_t z, T& rho, T (&u)[3], T (&ud)[3],
                                             T& uv) {
    const T x = vec[z * 3], y = vec[z * 3 + 1], w = vec[z * 3 + 2];
    rho = sqrt(x * x + y * y + w * w);
    const T inv = T(1) / rho;
    u[0] = x * inv; u[1] = y * inv; u[2] = w * inv;
    const T v0 = vdot[z * 3], v1 = vdot[z * 3 + 1], v2 = vdot[z * 3 + 2];
    uv = u[0] * v0 + u[1] * v1 + u[2] * v2;
    ud[0] = (v0 - uv * u[0]) * inv;
    ud[1] = (v1 - uv * u[1]) * inv;
    ud[2] = (v2 - uv * u[2]) * inv;
}

template <typename TAcc, int LMAX>
__global__ void __launch_bounds__(128) sh_jvp_kernel(int64_t E, const TAcc* __restrict__ vec, const TAcc* __restrict__ vdot, TAcc* __restrict__ Yd) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    __shared__ TAcc sY[128 * D];
    const int64_t z0 = (int64_t)blockIdx.x * 128;
    const int64_t z = z0 + threadIdx.x;
    if (z < E) {
        TAcc rho, u[3], ud[3], uv;
        unit_tangent(vec, vdot, z, rho, u, ud, uv);
        TAcc loc[D];
        sh_jvp<LMAX, TAcc>(u[0], u[1], u[2], ud[0], ud[1], ud[2], loc);
#pragma unroll
        for (int j = 0; j < D; ++j) sY[threadIdx.x * D + j] = loc[j];
    }
    __syncthreads();
    const int64_t n = min((int64_t)128, E - z0) * D;
    for (int64_t e = threadIdx.x; e < n; e += 128) Yd[z0 * D + e] = sY[e];
}

// f(r) = G(u), G = sum_k g_k Y_k:  grad f = (q - s u) / rho with q = grad G(u), s = u.q.  Its tangent:
//   (q_dot - s_dot u - s u_dot) / rho - (q - s u) (u.v) / rho^2,  q_dot = Hess G(u) u_dot,  s_dot = u_dot.q + u.q_dot
template <typename TAcc, int LMAX>
__global__ void __launch_bounds__(128) sh_hvp_kernel(int64_t E, const TAcc* __restrict__ vec, const TAcc* __restrict__ vdot,
                                                     const TAcc* __restrict__ gY, TAcc* __restrict__ gvec_dot) {
    constexpr int D = (LMAX + 1) * (LMAX + 1);
    __shared__ TAcc sG[128 * D];
    const int64_t z0 = (int64_t)blockIdx.x * 128;
    const int64_t n = min((int64_t)128, E - z0) * D;
    for (int64_t e = threadIdx.x; e < n; e += 128) sG[e] = gY[z0 * D + e];
    __syncthreads();
    const int64_t z = z0 + threadIdx.x;
    if (z >= E) return;
    TAcc rho, u[3], ud[3], uv;
    unit_tangent(vec, vdot, z, rho, u, ud, uv);
    TAcc g[D];
#pragma unroll
    for (int j = 0; j < D; ++j) g[j] = sG[threadIdx.x * D + j];
    TAcc q[3], qd[3];
    sh_grad<LMAX, TAcc>(u[0], u[1], u[2], g, q[0], q[1], q[2]);
    sh_hvp<LMAX, TAcc>(u[0], u[1], u[2], g, ud[0], ud[1], ud[2], qd[0], qd[1], qd[2]);
    const TAcc s = u[0] * q[0] + u[1] * q[1] + u[2] * q[2];
    const TAcc sd = ud[0] * q[0] + ud[1] * q[1] + ud[2] * q[2] + u[0] * qd[0] + u[1] * qd[1] + u[2] * qd[2];
    const TAcc inv = TAcc(1) / rho, c = uv * inv * inv;
#pragma unroll
    for (int a = 0; a < 3; ++a) gvec_dot[z * 3 + a] += (qd[a] - sd * u[a] - s * ud[a]) * inv - (q[a] - s * u[a]) * c;
}

// phi'' of the MLP nonlinearities (common.cuh holds phi and phi')
template <typename T>
__device__ __forceinline__ T d2silu_f(T x) {
    const T s = T(1) / (T(1) + ab2_exp(-x));
    return s * (T(1) - s) * (T(2) + x * (T(1) - T(2) * s));
}
// mish'' = (1 - t^2) sigma (2 + x (1 - sigma - 2 t sigma)), t = tanh(softplus(x)); the clamped x and the cancellation-free
// 1 - t^2 of dmish_f
template <typename T>
__device__ __forceinline__ T d2mish_f(T x) {
    const T xc = x < T(20) ? x : T(20);
    const T n = ab2_exp(xc), nn = n * (n + T(2)), d = nn + T(2);
    const T t = nn / d, omt2 = (T(2) / d) * (T(1) + t), sg = n / (T(1) + n);
    return omt2 * sg * (T(2) + xc * (T(1) - sg - T(2) * t * sg));
}
// gelu'' = pdf(x) (2 - x^2)
template <typename T>
__device__ __forceinline__ T d2gelu_f(T x) {
    return ab2_exp(T(-0.5) * x * x) * T(0.39894228040143267794) * (T(2) - x * x);
}
template <int NL, typename T>
__device__ __forceinline__ T d2act_f(T x) {
    if constexpr (NL == AB2_NL_MISH) return d2mish_f(x);
    else if constexpr (NL == AB2_NL_GELU) return d2gelu_f(x);
    else return d2silu_f(x);
}

template <typename TAct, typename TAcc, int NL>
__global__ void __launch_bounds__(256) act_bwd_jvp_kernel(int64_t n, const TAct* __restrict__ ga_dot, const TAct* __restrict__ ga,
                                                          const TAct* __restrict__ pre, const TAct* __restrict__ pre_dot,
                                                          TAct* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const TAcc x = to_acc<TAcc>(pre[i]);
    TAcc r = to_acc<TAcc>(ga[i]) * d2act_f<NL>(x) * to_acc<TAcc>(pre_dot[i]);
    if (ga_dot) r += to_acc<TAcc>(ga_dot[i]) * dact_f<NL>(x);
    out[i] = from_acc<TAct>(r);
}

template <typename T>
__device__ __forceinline__ T hvp_pow(T x, T p);
template <>
__device__ __forceinline__ float hvp_pow<float>(float x, float p) { return powf(x, p); }
template <>
__device__ __forceinline__ double hvp_pow<double>(double x, double p) { return pow(x, p); }

// e(r) = K A(r) / r with A = phi(s r) u(r / rmax), K = qq Z_i Z_j:  e' = K (A'/r - A/r^2), e'' = K (A''/r - 2A'/r^2 + 2A/r^3);
// the edge's Hessian applied to v is e'' (rh.v) rh + e'/r (v - (rh.v) rh)
template <typename T>
__global__ void __launch_bounds__(128) zbl_hvp_kernel(int64_t E, T p, T qq, const T* __restrict__ vec, const T* __restrict__ vdot,
                                                      const int32_t* __restrict__ ctr, const int32_t* __restrict__ nbr,
                                                      const int32_t* __restrict__ types, const T* __restrict__ Z,
                                                      const T* __restrict__ rmax_table, int num_types, T* __restrict__ gvec_dot) {
    const int64_t z = (int64_t)blockIdx.x * 128 + threadIdx.x;
    if (z >= E) return;
    const T vx = vec[3 * z], vy = vec[3 * z + 1], vz = vec[3 * z + 2];
    const T r = sqrt(vx * vx + vy * vy + vz * vz);
    const int tc = types[ctr[z]], tn = types[nbr[z]];
    const T zi = Z[tc], zj = Z[tn];
    const T rmax = rmax_table[tc * num_types + tn];
    const T x = r / rmax;
    if (!(x < T(1))) return;  // beyond the cutoff every term is exactly zero
    const T xp = hvp_pow(x, p);
    const T c0 = (p + T(1)) * (p + T(2)) / T(2), c1 = p * (p + T(2)), c2 = p * (p + T(1)) / T(2);
    const T u = T(1) - c0 * xp + c1 * xp * x - c2 * xp * x * x;
    const T du = (-c0 * p * xp / x + c1 * (p + T(1)) * xp - c2 * (p + T(2)) * xp * x) / rmax;
    const T d2u = (-c0 * p * (p - T(1)) * xp / (x * x) + c1 * (p + T(1)) * p * xp / x - c2 * (p + T(2)) * (p + T(1)) * xp) / (rmax * rmax);
    const T s = (hvp_pow(zi, T(0.23)) + hvp_pow(zj, T(0.23))) / T(0.46850);
    const T xs = s * r;
    const T e1 = T(0.02817) * ab2_exp(T(-0.20162) * xs), e2 = T(0.28022) * ab2_exp(T(-0.40290) * xs);
    const T e3 = T(0.50986) * ab2_exp(T(-0.94229) * xs), e4 = T(0.18175) * ab2_exp(T(-3.19980) * xs);
    const T phi = e1 + e2 + e3 + e4;
    const T dphi = s * (T(-0.20162) * e1 + T(-0.40290) * e2 + T(-0.94229) * e3 + T(-3.19980) * e4);
    const T d2phi = s * s * (T(0.20162 * 0.20162) * e1 + T(0.40290 * 0.40290) * e2 + T(0.94229 * 0.94229) * e3 + T(3.19980 * 3.19980) * e4);
    const T A = phi * u, dA = dphi * u + phi * du, d2A = d2phi * u + T(2) * dphi * du + phi * d2u;
    const T K = qq * zi * zj, ir = T(1) / r;
    const T de = K * (dA - A * ir) * ir;
    const T d2e = K * (d2A - T(2) * (dA - A * ir) * ir) * ir;
    const T ux = vx * ir, uy = vy * ir, uz = vz * ir;
    const T w0 = vdot[3 * z], w1 = vdot[3 * z + 1], w2 = vdot[3 * z + 2];
    const T uv = ux * w0 + uy * w1 + uz * w2;
    const T t = de * ir;
    gvec_dot[3 * z] += d2e * uv * ux + t * (w0 - uv * ux);
    gvec_dot[3 * z + 1] += d2e * uv * uy + t * (w1 - uv * uy);
    gvec_dot[3 * z + 2] += d2e * uv * uz + t * (w2 - uv * uz);
}

}  // namespace

extern "C" int ab2_sh_jvp(int acc_dtype, int lmax, int64_t E, const void* vec, const void* vdot, void* Yd, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "edge vectors must be fp64 or fp32");
    AB2_CHECK_ARG(vec && vdot && Yd, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, AB2_DISPATCH_LMAX(lmax, sh_jvp_kernel<TAcc, LMAX><<<ab2_blocks(E, 128), 128, 0, st>>>(
                                                            E, (const TAcc*)vec, (const TAcc*)vdot, (TAcc*)Yd)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_sh_hvp(int acc_dtype, int lmax, int64_t E, const void* vec, const void* vdot, const void* gY, void* gvec_dot,
                          void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "edge vectors must be fp64 or fp32");
    AB2_CHECK_ARG(vec && vdot && gY && gvec_dot, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_ACC(acc_dtype, AB2_DISPATCH_LMAX(lmax, sh_hvp_kernel<TAcc, LMAX><<<ab2_blocks(E, 128), 128, 0, st>>>(
                                                            E, (const TAcc*)vec, (const TAcc*)vdot, (const TAcc*)gY, (TAcc*)gvec_dot)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_act_bwd_jvp(int dtype, int64_t n, const void* ga_dot, const void* ga, const void* pre, const void* pre_dot, void* out,
                               int nonlin, void* stream) {
    AB2_CHECK_ARG(nonlin == AB2_NL_SILU || nonlin == AB2_NL_MISH || nonlin == AB2_NL_GELU, "nonlinearity");
    AB2_CHECK_ARG(n >= 0, "sizes");
    if (n == 0) return 0;
    AB2_CHECK_ARG(ga && pre && pre_dot && out, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_NL(nonlin, AB2_DISPATCH_DTYPE(dtype, act_bwd_jvp_kernel<TAct, TAcc, NL><<<ab2_blocks(n, 256), 256, 0, st>>>(
                                                          n, (const TAct*)ga_dot, (const TAct*)ga, (const TAct*)pre, (const TAct*)pre_dot,
                                                          (TAct*)out)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_zbl_hvp(int acc_dtype, int64_t E, int num_types, double p_cut, double qq, const void* vec, const void* vdot,
                           const int32_t* ctr, const int32_t* nbr, const int32_t* types, const void* Z, const void* rmax_table,
                           void* gvec_dot, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "ab2_zbl_hvp works in the accumulate type (fp32 / fp64)");
    AB2_CHECK_ARG(vec && vdot && ctr && nbr && types && Z && rmax_table && gvec_dot && num_types > 0, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (acc_dtype == AB2_F64)
        zbl_hvp_kernel<double><<<ab2_blocks(E, 128), 128, 0, st>>>(E, p_cut, qq, (const double*)vec, (const double*)vdot, ctr, nbr, types,
                                                                  (const double*)Z, (const double*)rmax_table, num_types, (double*)gvec_dot);
    else
        zbl_hvp_kernel<float><<<ab2_blocks(E, 128), 128, 0, st>>>(E, (float)p_cut, (float)qq, (const float*)vec, (const float*)vdot, ctr, nbr,
                                                                 types, (const float*)Z, (const float*)rmax_table, num_types, (float*)gvec_dot);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// Radial basis of the two-body scalar embedding (BesselEdgeLengthEncoding + PolynomialCutoff,
// allegro/nn/scalarembed.py:60-66), shared by the radial kernels (radial.cu) and the fused gradient GEMM + radial
// adjoint (linear_tc.cu):
//
//   B_n(x) = sin(pi w_n x)/(pi x) * f_p(x),   x = |r| / r_max(t_c, t_n),   zero for x >= 1
#pragma once

#include "common.cuh"

#define AB2_MAX_BESSEL 16

template <typename T>
__device__ __forceinline__ T ab2_sin(T x);
template <>
__device__ __forceinline__ float ab2_sin<float>(float x) { return sinf(x); }
template <>
__device__ __forceinline__ double ab2_sin<double>(double x) { return sin(x); }
template <typename T>
__device__ __forceinline__ T ab2_cos(T x);
template <>
__device__ __forceinline__ float ab2_cos<float>(float x) { return cosf(x); }
template <>
__device__ __forceinline__ double ab2_cos<double>(double x) { return cos(x); }
__device__ __forceinline__ float ab2_pow(float x, float p) { return powf(x, p); }
__device__ __forceinline__ double ab2_pow(double x, double p) { return pow(x, p); }

// radial basis and (optionally) its derivative w.r.t. x
template <typename TAcc, bool GRAD>
__device__ __forceinline__ void bessel_basis(TAcc x, TAcc p, int nb, const TAcc* __restrict__ bw, TAcc* B, TAcc* dB) {
    const TAcc PI = TAcc(3.14159265358979323846);
    if (x >= TAcc(1)) {
        for (int n = 0; n < nb; ++n) {
            B[n] = TAcc(0);
            if (GRAD) dB[n] = TAcc(0);
        }
        return;
    }
    const TAcc xp = ab2_pow(x, p);  // x^p
    const TAcc a = (p + 1) * (p + 2) / 2, b = p * (p + 2), c = p * (p + 1) / 2;
    const TAcc f = TAcc(1) - a * xp + b * xp * x - c * xp * x * x;
    const TAcc df = GRAD ? (-a * p * xp / x + b * (p + 1) * xp - c * (p + 2) * xp * x) : TAcc(0);
    const TAcc inv = TAcc(1) / (PI * x);
    for (int n = 0; n < nb; ++n) {
        const TAcc arg = PI * bw[n] * x;
        const TAcc s = ab2_sin(arg) * inv;  // sin(pi w x)/(pi x)
        B[n] = s * f;
        if (GRAD) {
            const TAcc ds = (bw[n] * ab2_cos(arg) - s) / x;  // d/dx [sin(pi w x)/(pi x)]
            dB[n] = ds * f + s * df;
        }
    }
}

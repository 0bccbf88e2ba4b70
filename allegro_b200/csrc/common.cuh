// Shared helpers for the allegro_b200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstring>

#include "../../include/allegro_b200.h"

// ---------------------------------------------------------------------------------------
// error plumbing (thread-local message, returned through ab2_last_error)
// ---------------------------------------------------------------------------------------
void ab2_set_error(const char* fmt, ...);

#define AB2_CHECK_ARG(cond, msg)                                                       \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            ab2_set_error("%s:%d: bad argument: %s (%s)", __FILE__, __LINE__, msg, #cond); \
            return 1;                                                                  \
        }                                                                              \
    } while (0)

#define AB2_CUDA_LAUNCH_CHECK()                                                        \
    do {                                                                               \
        cudaError_t e__ = cudaGetLastError();                                          \
        if (e__ != cudaSuccess) {                                                      \
            ab2_set_error("%s:%d: CUDA launch failed: %s", __FILE__, __LINE__,         \
                          cudaGetErrorString(e__));                                    \
            return 2;                                                                  \
        }                                                                              \
    } while (0)

#define AB2_CUDA_CALL(x)                                                               \
    do {                                                                               \
        cudaError_t e__ = (x);                                                         \
        if (e__ != cudaSuccess) {                                                      \
            ab2_set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #x,              \
                          cudaGetErrorString(e__));                                    \
            return 2;                                                                  \
        }                                                                              \
    } while (0)

// ---------------------------------------------------------------------------------------
// dtype dispatch:  TAct = storage type of activations, TAcc = accumulation type
// ---------------------------------------------------------------------------------------
typedef __nv_bfloat16 bf16;

#define AB2_DISPATCH_DTYPE(dtype, ...)                                                 \
    switch (dtype) {                                                                   \
        case AB2_F64: {                                                                \
            using TAct = double;                                                       \
            using TAcc = double;                                                       \
            __VA_ARGS__;                                                               \
        } break;                                                                       \
        case AB2_F32: {                                                                \
            using TAct = float;                                                        \
            using TAcc = float;                                                        \
            __VA_ARGS__;                                                               \
        } break;                                                                       \
        case AB2_BF16: {                                                               \
            using TAct = bf16;                                                         \
            using TAcc = float;                                                        \
            __VA_ARGS__;                                                               \
        } break;                                                                       \
        default:                                                                       \
            ab2_set_error("unknown dtype %d", (int)(dtype));                           \
            return 1;                                                                  \
    }

// accumulate-type-only dispatch (geometry / energies)
#define AB2_DISPATCH_ACC(dtype, ...)                                                   \
    switch (dtype) {                                                                   \
        case AB2_F64: {                                                                \
            using TAcc = double;                                                       \
            __VA_ARGS__;                                                               \
        } break;                                                                       \
        case AB2_F32:                                                                  \
        case AB2_BF16: {                                                               \
            using TAcc = float;                                                        \
            __VA_ARGS__;                                                               \
        } break;                                                                       \
        default:                                                                       \
            ab2_set_error("unknown dtype %d", (int)(dtype));                           \
            return 1;                                                                  \
    }

#define AB2_DISPATCH_LMAX(lmax, ...)                                                   \
    switch (lmax) {                                                                    \
        case 0: { constexpr int LMAX = 0; __VA_ARGS__; } break;                        \
        case 1: { constexpr int LMAX = 1; __VA_ARGS__; } break;                        \
        case 2: { constexpr int LMAX = 2; __VA_ARGS__; } break;                        \
        case 3: { constexpr int LMAX = 3; __VA_ARGS__; } break;                        \
        case 4: { constexpr int LMAX = 4; __VA_ARGS__; } break;                        \
        default:                                                                       \
            ab2_set_error("lmax %d not supported (max %d)", (int)(lmax), AB2_MAX_LMAX); \
            return 1;                                                                  \
    }

template <typename TAcc, typename T>
__device__ __forceinline__ TAcc to_acc(T v) { return (TAcc)v; }
template <>
__device__ __forceinline__ float to_acc<float, bf16>(bf16 v) { return __bfloat162float(v); }

template <typename T, typename TAcc>
__device__ __forceinline__ T from_acc(TAcc v) { return (T)v; }
template <>
__device__ __forceinline__ bf16 from_acc<bf16, float>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float ab2_exp(float x) { return expf(x); }
__device__ __forceinline__ double ab2_exp(double x) { return exp(x); }

template <typename T>
__device__ __forceinline__ T silu_f(T x) { return x / (T(1) + ab2_exp(-x)); }
template <typename T>
__device__ __forceinline__ T dsilu_f(T x) {
    T s = T(1) / (T(1) + ab2_exp(-x));
    return s * (T(1) + x * (T(1) - s));
}

__device__ __forceinline__ float ab2_erfc(float x) { return erfcf(x); }
__device__ __forceinline__ double ab2_erfc(double x) { return erfc(x); }

// mish(x) = x tanh(softplus(x)).  With n = e^min(x, 20): tanh(softplus(x)) = n (n + 2) / (n (n + 2) + 2), and 1 - tanh =
// 2 / (n (n + 2) + 2) without cancellation; past x = 20 the clamp changes tanh by less than 1e-17.
template <typename T>
__device__ __forceinline__ T mish_f(T x) {
    const T n = ab2_exp(x < T(20) ? x : T(20)), nn = n * (n + T(2));
    return x * (nn / (nn + T(2)));
}
// mish'(x) = t + x (1 - t^2) sigma(x), t = tanh(softplus(x)), sigma(x) = n / (1 + n).  The second term takes the clamped
// x as well: past 20 it is below 4e-16 (true and clamped), where the unclamped x times the clamped 1 - t^2 would grow with x.
template <typename T>
__device__ __forceinline__ T dmish_f(T x) {
    const T xc = x < T(20) ? x : T(20);
    const T n = ab2_exp(xc), nn = n * (n + T(2)), d = nn + T(2);
    const T t = nn / d, omt = T(2) / d;
    return t + xc * (omt * (T(1) + t)) * (n / (T(1) + n));
}
// gelu(x) = x Phi(x) = x erfc(-x / sqrt2) / 2, the exact (erf) form; erfc instead of 1 + erf, which cancels for x < -3
template <typename T>
__device__ __forceinline__ T gelu_f(T x) { return T(0.5) * x * ab2_erfc(-x * T(0.70710678118654752440)); }
template <typename T>
__device__ __forceinline__ T dgelu_f(T x) {
    return T(0.5) * ab2_erfc(-x * T(0.70710678118654752440)) + x * ab2_exp(T(-0.5) * x * x) * T(0.39894228040143267794);
}

// the MLP nonlinearity NL (AB2_NL_*) and its derivative, in T = float / double
template <int NL, typename T>
__device__ __forceinline__ T act_f(T x) {
    if constexpr (NL == AB2_NL_MISH) return mish_f(x);
    else if constexpr (NL == AB2_NL_GELU) return gelu_f(x);
    else return silu_f(x);
}
template <int NL, typename T>
__device__ __forceinline__ T dact_f(T x) {
    if constexpr (NL == AB2_NL_MISH) return dmish_f(x);
    else if constexpr (NL == AB2_NL_GELU) return dgelu_f(x);
    else return dsilu_f(x);
}

// nonlinearity dispatch: NL = the constexpr AB2_NL_* code
#define AB2_DISPATCH_NL(nonlin, ...)                                                   \
    switch (nonlin) {                                                                  \
        case AB2_NL_SILU: { constexpr int NL = AB2_NL_SILU; __VA_ARGS__; } break;      \
        case AB2_NL_MISH: { constexpr int NL = AB2_NL_MISH; __VA_ARGS__; } break;      \
        case AB2_NL_GELU: { constexpr int NL = AB2_NL_GELU; __VA_ARGS__; } break;      \
        default:                                                                       \
            ab2_set_error("unknown nonlinearity %d", (int)(nonlin));                   \
            return 1;                                                                  \
    }

// irrep (l) of SH component j: floor(sqrt(j)) for j < 25
__host__ __device__ __forceinline__ int sh_l_of(int j) { return (j >= 16) ? 4 : (j >= 9) ? 3 : (j >= 4) ? 2 : (j >= 1) ? 1 : 0; }

// a * b + c per component (two FFMA on sm_90: Hopper has no paired FP32 FMA)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Reduce D (<=16) per-lane values across the warp with a multi-value butterfly: 16 shuffles instead
// of 5*D.  On return lane 2*j (and 2*j+1) holds the warp total of value j.
template <typename TAcc, int D>
__device__ __forceinline__ TAcc warp_multi_sum(const TAcc (&v)[D], int lane) {
    static_assert(D <= 16, "at most 16 values");
    TAcc a[16];
#pragma unroll
    for (int t = 0; t < 16; ++t) a[t] = t < D ? v[t] : TAcc(0);
    TAcc b[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
        const bool up = lane & 16;
        const TAcc send = up ? a[t] : a[t + 8];
        const TAcc got = __shfl_xor_sync(0xffffffffu, send, 16);
        b[t] = (up ? a[t + 8] : a[t]) + got;
    }
    TAcc c[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        const bool up = lane & 8;
        const TAcc send = up ? b[t] : b[t + 4];
        const TAcc got = __shfl_xor_sync(0xffffffffu, send, 8);
        c[t] = (up ? b[t + 4] : b[t]) + got;
    }
    TAcc d[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
        const bool up = lane & 4;
        const TAcc send = up ? c[t] : c[t + 2];
        const TAcc got = __shfl_xor_sync(0xffffffffu, send, 4);
        d[t] = (up ? c[t + 2] : c[t]) + got;
    }
    const bool up = lane & 2;
    const TAcc send = up ? d[0] : d[1];
    const TAcc got = __shfl_xor_sync(0xffffffffu, send, 2);
    TAcc e = (up ? d[1] : d[0]) + got;
    e += __shfl_xor_sync(0xffffffffu, e, 1);
    return e;  // value index = lane >> 1
}

static inline unsigned ab2_blocks(int64_t n, int per) { return (unsigned)((n + per - 1) / per); }

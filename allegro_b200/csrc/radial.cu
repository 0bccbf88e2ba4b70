// Upstream two-body scalar track (SURVEY section 8 row f1) and edge geometry, so that the whole
// energy+force evaluation runs without torch autograd:
//
//   edge vectors      r_z = pos[nbr] - pos[ctr] (+ shift)          nequip with_edge_vectors_ (tensorembed.py:86)
//   x = |r| / r_max(t_c, t_n)                                      EdgeLengthNormalizer (allegro_models.py:153-157)
//   B_n(x) = sin(pi w_n x)/(pi x) * f_p(x),  n = 1..num_bessels    BesselEdgeLengthEncoding + PolynomialCutoff
//                                                                  (allegro/nn/scalarembed.py:60-66)
//   e0[z][c] = typeemb[t_c, t_n][c] * sum_n B_n W_b[n][c]          ProductTypeEmbedding (_edgeembed.py:68-85)
//
// and the adjoint (g_e0 -> d/d r_z); nothing but e0 / g_e0 touches HBM.
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

template <typename TPos, typename TAcc>
__global__ void __launch_bounds__(256) edge_vec_kernel(int64_t E, const TPos* __restrict__ pos, const int32_t* __restrict__ ctr,
                                                       const int32_t* __restrict__ nbr, const TPos* __restrict__ shift,
                                                       TAcc* __restrict__ vec) {
    const int64_t z = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (z >= E) return;
    const int64_t i = ctr[z], j = nbr[z];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        TPos d = pos[j * 3 + a] - pos[i * 3 + a];
        if (shift) d += shift[z * 3 + a];
        vec[z * 3 + a] = (TAcc)d;
    }
}

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

// Block = 256 edges.  Phase 1: one thread per edge evaluates the radial basis ONCE (sin/pow are the
// expensive part) into shared memory.  Phase 2: one warp per edge, lane = embedding column(s), so the
// [E][S_rc] rows are written (read) with coalesced 128-byte accesses.
template <typename TAct, typename TAcc>
__global__ void __launch_bounds__(256) radial_fwd_kernel(int64_t E, int S_rc, int nb, TAcc p, const TAcc* __restrict__ vec,
                                                         const int32_t* __restrict__ ctr, const int32_t* __restrict__ nbr,
                                                         const int32_t* __restrict__ types, const TAcc* __restrict__ rmax_table,
                                                         int num_types, const TAcc* __restrict__ bw, const TAcc* __restrict__ Wb,
                                                         const TAcc* __restrict__ cemb, const TAcc* __restrict__ nemb,
                                                         TAct* __restrict__ e0) {
    __shared__ TAcc sB[AB2_MAX_BESSEL][256];
    __shared__ int s_tc[256], s_tn[256];
    const int t = threadIdx.x;
    const int64_t z0 = (int64_t)blockIdx.x * 256;
    {
        const int64_t z = z0 + t;
        TAcc B[AB2_MAX_BESSEL];
        int tc = 0, tn = 0;
        if (z < E) {
            const TAcc vx = vec[z * 3], vy = vec[z * 3 + 1], vz = vec[z * 3 + 2];
            const TAcc r = sqrt(vx * vx + vy * vy + vz * vz);
            tc = types[ctr[z]];
            tn = types[nbr[z]];
            bessel_basis<TAcc, false>(r / rmax_table[tc * num_types + tn], p, nb, bw, B, nullptr);
        } else {
            for (int n = 0; n < nb; ++n) B[n] = TAcc(0);
        }
        for (int n = 0; n < nb; ++n) sB[n][t] = B[n];
        s_tc[t] = tc;
        s_tn[t] = tn;
    }
    __syncthreads();
    const int warp = t >> 5, lane = t & 31, half = S_rc >> 1;
    for (int e = warp; e < 256; e += 8) {
        const int64_t z = z0 + e;
        if (z >= E) break;
        const int tc = s_tc[e], tn = s_tn[e];
        for (int c = lane; c < S_rc; c += 32) {
            TAcc s = TAcc(0);
            for (int n = 0; n < nb; ++n) s += sB[n][e] * Wb[n * S_rc + c];
            const TAcc te = (c < half) ? cemb[tc * half + c] : nemb[tn * half + (c - half)];
            e0[z * S_rc + c] = from_acc<TAct>(te * s);
        }
    }
}

template <typename TAct, typename TAcc>
__global__ void __launch_bounds__(256) radial_bwd_kernel(int64_t E, int S_rc, int nb, TAcc p, const TAcc* __restrict__ vec,
                                                         const int32_t* __restrict__ ctr, const int32_t* __restrict__ nbr,
                                                         const int32_t* __restrict__ types, const TAcc* __restrict__ rmax_table,
                                                         int num_types, const TAcc* __restrict__ bw, const TAcc* __restrict__ Wb,
                                                         const TAcc* __restrict__ cemb, const TAcc* __restrict__ nemb,
                                                         const TAct* __restrict__ ge0, TAcc* __restrict__ gvec) {
    __shared__ TAcc sdB[AB2_MAX_BESSEL][256];
    __shared__ TAcc s_gx[256];
    __shared__ int s_tc[256], s_tn[256];
    const int t = threadIdx.x;
    const int64_t z0 = (int64_t)blockIdx.x * 256;
    const int64_t zt = z0 + t;
    TAcc vx = 0, vy = 0, vz = 0, r = 1, rmax = 1;
    {
        TAcc B[AB2_MAX_BESSEL], dB[AB2_MAX_BESSEL];
        int tc = 0, tn = 0;
        if (zt < E) {
            vx = vec[zt * 3]; vy = vec[zt * 3 + 1]; vz = vec[zt * 3 + 2];
            r = sqrt(vx * vx + vy * vy + vz * vz);
            tc = types[ctr[zt]];
            tn = types[nbr[zt]];
            rmax = rmax_table[tc * num_types + tn];
            bessel_basis<TAcc, true>(r / rmax, p, nb, bw, B, dB);
        } else {
            for (int n = 0; n < nb; ++n) dB[n] = TAcc(0);
        }
        for (int n = 0; n < nb; ++n) sdB[n][t] = dB[n];
        s_tc[t] = tc;
        s_tn[t] = tn;
    }
    __syncthreads();
    // gx = sum_c ge0[c] te[c] (sum_n dB[n] Wb[n][c])
    const int warp = t >> 5, lane = t & 31, half = S_rc >> 1;
    for (int e = warp; e < 256; e += 8) {
        const int64_t z = z0 + e;
        if (z >= E) break;
        const int tc = s_tc[e], tn = s_tn[e];
        TAcc gx = TAcc(0);
        for (int c = lane; c < S_rc; c += 32) {
            TAcc s = TAcc(0);
            for (int n = 0; n < nb; ++n) s += sdB[n][e] * Wb[n * S_rc + c];
            const TAcc te = (c < half) ? cemb[tc * half + c] : nemb[tn * half + (c - half)];
            gx += to_acc<TAcc>(ge0[z * S_rc + c]) * te * s;
        }
        gx = warp_sum(gx);
        if (lane == 0) s_gx[e] = gx;
    }
    __syncthreads();
    if (zt < E) {
        const TAcc f = s_gx[t] / (rmax * r);  // dx/dr_vec = r_vec / (|r| r_max)
        gvec[zt * 3] += f * vx;
        gvec[zt * 3 + 1] += f * vy;
        gvec[zt * 3 + 2] += f * vz;
    }
}

extern "C" int ab2_edge_vec(int pos_dtype, int acc_dtype, int64_t E, const void* pos, const int32_t* ctr, const int32_t* nbr,
                            const void* shift, void* vec, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(pos && ctr && nbr && vec, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned g = ab2_blocks(E, 256);
    const bool acc64 = acc_dtype == AB2_F64;
    if (pos_dtype == AB2_F64 && acc64)
        edge_vec_kernel<double, double><<<g, 256, 0, st>>>(E, (const double*)pos, ctr, nbr, (const double*)shift, (double*)vec);
    else if (pos_dtype == AB2_F64)
        edge_vec_kernel<double, float><<<g, 256, 0, st>>>(E, (const double*)pos, ctr, nbr, (const double*)shift, (float*)vec);
    else if (acc64)
        edge_vec_kernel<float, double><<<g, 256, 0, st>>>(E, (const float*)pos, ctr, nbr, (const float*)shift, (double*)vec);
    else
        edge_vec_kernel<float, float><<<g, 256, 0, st>>>(E, (const float*)pos, ctr, nbr, (const float*)shift, (float*)vec);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_radial_fwd(int dtype, int64_t E, int S_rc, int num_bessels, double p_cut, const void* vec, const int32_t* ctr,
                              const int32_t* nbr, const int32_t* types, const void* rmax_table, int num_types, const void* bessel_w,
                              const void* Wb, const void* center_embed, const void* neighbor_embed, void* e0, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(vec && ctr && nbr && types && rmax_table && bessel_w && Wb && center_embed && neighbor_embed && e0, "null pointer");
    AB2_CHECK_ARG(num_bessels > 0 && num_bessels <= AB2_MAX_BESSEL && S_rc > 0 && S_rc % 2 == 0, "num_bessels / embedding dim");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_DTYPE(dtype, radial_fwd_kernel<TAct, TAcc><<<ab2_blocks(E, 256), 256, 0, st>>>(
                                  E, S_rc, num_bessels, (TAcc)p_cut, (const TAcc*)vec, ctr, nbr, types, (const TAcc*)rmax_table, num_types,
                                  (const TAcc*)bessel_w, (const TAcc*)Wb, (const TAcc*)center_embed, (const TAcc*)neighbor_embed, (TAct*)e0));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_radial_bwd(int dtype, int64_t E, int S_rc, int num_bessels, double p_cut, const void* vec, const int32_t* ctr,
                              const int32_t* nbr, const int32_t* types, const void* rmax_table, int num_types, const void* bessel_w,
                              const void* Wb, const void* center_embed, const void* neighbor_embed, const void* g_e0, void* gvec,
                              void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(vec && ctr && nbr && types && rmax_table && bessel_w && Wb && center_embed && neighbor_embed && g_e0 && gvec, "null pointer");
    AB2_CHECK_ARG(num_bessels > 0 && num_bessels <= AB2_MAX_BESSEL && S_rc > 0 && S_rc % 2 == 0, "num_bessels / embedding dim");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_DTYPE(dtype, radial_bwd_kernel<TAct, TAcc><<<ab2_blocks(E, 256), 256, 0, st>>>(
                                  E, S_rc, num_bessels, (TAcc)p_cut, (const TAcc*)vec, ctr, nbr, types, (const TAcc*)rmax_table, num_types,
                                  (const TAcc*)bessel_w, (const TAcc*)Wb, (const TAcc*)center_embed, (const TAcc*)neighbor_embed,
                                  (const TAct*)g_e0, (TAcc*)gvec));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// ---------------------------------------------------------------------------------------
// Radial embedding with per-type-pair matrices ("PQ" form), forward and adjoint:
//
//     out[z][c] = sum_n B_n(x_z) * PQ[t_c * T + t_n][n][c]
//
// The reference's product embedding (allegro/nn/_edgeembed.py:68-85) is the case PQ = typeemb(t_c,t_n)[c] * W_b[n][c];
// since everything between the radial basis and the first nonlinearity is LINEAR (type-embedding product, first layer
// of scalar_embed_mlp, allegro_models.py:153-183) the host can also fold that layer's weights in,
//     PQ[t_c,t_n] = W_b diag(typeemb(t_c,t_n)) W_1        (nb x width),
// and this kernel then emits the MLP's first pre-activation directly: the [E][S] embedding tensor and one GEMM per
// direction disappear.  Structure: 256 edges per block; phase 1 one thread per edge evaluates the basis (and its
// derivative) once into shared memory; phase 2 one warp per 32 CONSECUTIVE edges, lane = output column(s), the
// nb x CPL matrix slice of the current type pair held in registers (reloaded only when the pair changes -- never for a
// single-species system), so an edge costs nb*CPL FMAs + CPL coalesced stores.
// ---------------------------------------------------------------------------------------
template <typename TAct, typename TAcc, int NB, int CPL>
__global__ void __launch_bounds__(256) radial_pq_fwd_kernel(int64_t E, int S, TAcc p, const TAcc* __restrict__ vec,
                                                            const int32_t* __restrict__ ctr, const int32_t* __restrict__ nbr,
                                                            const int32_t* __restrict__ types, const TAcc* __restrict__ rmax_table,
                                                            int num_types, const TAcc* __restrict__ bw, const TAcc* __restrict__ PQ,
                                                            TAct* __restrict__ out) {
    __shared__ TAcc sB[NB][256];
    __shared__ int s_pair[256];
    const int t = threadIdx.x;
    const int64_t z0 = (int64_t)blockIdx.x * 256;
    {
        const int64_t z = z0 + t;
        TAcc B[NB];
        int pair = 0;
        if (z < E) {
            const TAcc vx = vec[z * 3], vy = vec[z * 3 + 1], vz = vec[z * 3 + 2];
            const TAcc r = sqrt(vx * vx + vy * vy + vz * vz);
            const int tc = types[ctr[z]], tn = types[nbr[z]];
            pair = tc * num_types + tn;
            bessel_basis<TAcc, false>(r / rmax_table[pair], p, NB, bw, B, nullptr);
        } else {
#pragma unroll
            for (int n = 0; n < NB; ++n) B[n] = TAcc(0);
        }
#pragma unroll
        for (int n = 0; n < NB; ++n) sB[n][t] = B[n];
        s_pair[t] = pair;
    }
    __syncthreads();
    const int warp = t >> 5, lane = t & 31;
    TAcc m[NB][CPL];
    int cur = -1;
    for (int e = warp * 32; e < warp * 32 + 32; ++e) {
        const int64_t z = z0 + e;
        if (z >= E) break;
        const int pair = s_pair[e];
        if (pair != cur) {  // warp-uniform
            cur = pair;
#pragma unroll
            for (int n = 0; n < NB; ++n)
#pragma unroll
                for (int q = 0; q < CPL; ++q) m[n][q] = (lane + 32 * q < S) ? PQ[((int64_t)pair * NB + n) * S + lane + 32 * q] : TAcc(0);
        }
        TAcc acc[CPL];
#pragma unroll
        for (int q = 0; q < CPL; ++q) acc[q] = TAcc(0);
#pragma unroll
        for (int n = 0; n < NB; ++n) {
            const TAcc b = sB[n][e];
#pragma unroll
            for (int q = 0; q < CPL; ++q) acc[q] += b * m[n][q];
        }
#pragma unroll
        for (int q = 0; q < CPL; ++q)
            if (lane + 32 * q < S) out[z * S + lane + 32 * q] = from_acc<TAct>(acc[q]);
    }
}

// adjoint: gvec[z] += d out / d vec ^T (g_out[z] (* silu'(aux[z]) if aux)).
// ONE THREAD PER EDGE end to end: gx = sum_c g[c] * sum_n dB_n * PQ[pair][n][c] needs no cross-lane reduction when the
// thread walks its own row (S contiguous values, 16-byte loads, all independent -> deep memory-level parallelism),
// and the PQ entries are warp-uniform broadcasts (same type pair for most lanes; L1-resident 2-4 KB per pair).
// The first version (warp per edge, lane = column) serialised 32 edges per warp behind a load -> shuffle-reduce chain.
template <typename TAct, typename TAcc, int NB, int CPL>
__global__ void __launch_bounds__(128) radial_pq_bwd_kernel(int64_t E, int S, TAcc p, const TAcc* __restrict__ vec,
                                                            const int32_t* __restrict__ ctr, const int32_t* __restrict__ nbr,
                                                            const int32_t* __restrict__ types, const TAcc* __restrict__ rmax_table,
                                                            int num_types, const TAcc* __restrict__ bw, const TAcc* __restrict__ PQ,
                                                            const TAct* __restrict__ g_out, const TAct* __restrict__ aux,
                                                            TAcc* __restrict__ gvec) {
    const int64_t z = (int64_t)blockIdx.x * 128 + threadIdx.x;
    if (z >= E) return;
    const TAcc vx = vec[z * 3], vy = vec[z * 3 + 1], vz = vec[z * 3 + 2];
    const TAcc r = sqrt(vx * vx + vy * vy + vz * vz);
    const int pair = types[ctr[z]] * num_types + types[nbr[z]];
    const TAcc rmax = rmax_table[pair];
    TAcc B[NB], dB[NB];
    bessel_basis<TAcc, true>(r / rmax, p, NB, bw, B, dB);
    const TAcc* __restrict__ m = PQ + (int64_t)pair * NB * S;
    const TAct* __restrict__ g = g_out + z * S;
    const TAct* __restrict__ a = aux ? aux + z * S : nullptr;
    TAcc gx = TAcc(0);
    constexpr int V = 16 / (int)sizeof(TAct);  // elements per 16-byte load
    if (S % V == 0) {
        for (int c0 = 0; c0 < S; c0 += V) {
            TAct gv[V], av[V];
            *reinterpret_cast<uint4*>(gv) = *reinterpret_cast<const uint4*>(g + c0);
            if (a) *reinterpret_cast<uint4*>(av) = *reinterpret_cast<const uint4*>(a + c0);
#pragma unroll
            for (int k = 0; k < V; ++k) {
                TAcc gc = to_acc<TAcc>(gv[k]);
                if (a) gc *= dsilu_f(to_acc<TAcc>(av[k]));
                TAcc sN = TAcc(0);
#pragma unroll
                for (int n = 0; n < NB; ++n) sN += dB[n] * __ldg(m + n * S + c0 + k);
                gx += gc * sN;
            }
        }
    } else {
        for (int c = 0; c < S; ++c) {
            TAcc gc = to_acc<TAcc>(g[c]);
            if (a) gc *= dsilu_f(to_acc<TAcc>(a[c]));
            TAcc sN = TAcc(0);
#pragma unroll
            for (int n = 0; n < NB; ++n) sN += dB[n] * __ldg(m + n * S + c);
            gx += gc * sN;
        }
    }
    const TAcc f = gx / (rmax * r);  // dx/dr_vec = r_vec / (|r| r_max)
    gvec[z * 3] += f * vx;
    gvec[z * 3 + 1] += f * vy;
    gvec[z * 3 + 2] += f * vz;
}

// (A warp-cooperative variant -- 32-column chunks moved with row-contiguous 128-byte segments through a padded shared-memory
// tile, then the same row walk -- is slower: the tile's load -> silu' -> store -> sync -> load chain with 16 resident warps
// hides less latency than 32 independent 16-byte loads per thread with 32+ resident warps, uncoalesced as they are.)

#define AB2_RADIAL_PQ_DISPATCH(KERNEL, ...)                                                                       \
    do {                                                                                                          \
        const int cpl = (S + 31) / 32;                                                                            \
        if (cpl == 1) { AB2_DISPATCH_DTYPE(dtype, KERNEL<TAct, TAcc, 8, 1><<<ab2_blocks(E, 256), 256, 0, st>>>(__VA_ARGS__)); } \
        else if (cpl == 2) { AB2_DISPATCH_DTYPE(dtype, KERNEL<TAct, TAcc, 8, 2><<<ab2_blocks(E, 256), 256, 0, st>>>(__VA_ARGS__)); } \
        else { AB2_DISPATCH_DTYPE(dtype, KERNEL<TAct, TAcc, 8, 4><<<ab2_blocks(E, 256), 256, 0, st>>>(__VA_ARGS__)); } \
    } while (0)

extern "C" int ab2_radial_pq_fwd(int dtype, int64_t E, int S, int num_bessels, double p_cut, const void* vec, const int32_t* ctr,
                                 const int32_t* nbr, const int32_t* types, const void* rmax_table, int num_types, const void* bessel_w,
                                 const void* PQ, void* out, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(vec && ctr && nbr && types && rmax_table && bessel_w && PQ && out, "null pointer");
    AB2_CHECK_ARG(num_bessels == 8 && S > 0 && S <= 128, "radial_pq: 8 Bessel functions, at most 128 output columns");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_RADIAL_PQ_DISPATCH(radial_pq_fwd_kernel, E, S, (TAcc)p_cut, (const TAcc*)vec, ctr, nbr, types, (const TAcc*)rmax_table, num_types,
                           (const TAcc*)bessel_w, (const TAcc*)PQ, (TAct*)out);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_radial_pq_bwd(int dtype, int64_t E, int S, int num_bessels, double p_cut, const void* vec, const int32_t* ctr,
                                 const int32_t* nbr, const int32_t* types, const void* rmax_table, int num_types, const void* bessel_w,
                                 const void* PQ, const void* g_out, const void* aux, void* gvec, void* stream) {
    if (E == 0) return 0;
    AB2_CHECK_ARG(vec && ctr && nbr && types && rmax_table && bessel_w && PQ && g_out && gvec, "null pointer");
    AB2_CHECK_ARG(num_bessels == 8 && S > 0 && S <= 128, "radial_pq: 8 Bessel functions, at most 128 output columns");
    cudaStream_t st = (cudaStream_t)stream;
    AB2_DISPATCH_DTYPE(dtype, radial_pq_bwd_kernel<TAct, TAcc, 8, 1><<<ab2_blocks(E, 128), 128, 0, st>>>(
                                  E, S, (TAcc)p_cut, (const TAcc*)vec, ctr, nbr, types, (const TAcc*)rmax_table, num_types, (const TAcc*)bessel_w,
                                  (const TAcc*)PQ, (const TAct*)g_out, (const TAct*)aux, (TAcc*)gvec));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// Fused linear layer of the scalar track (nequip ScalarMLPFunction layers used at
// /root/reference/allegro/nn/_allegro.py:251,278, tensorembed.py:88-89, allegro_models.py:231-241).
//
//   Out[M][N] (+)= epi( act( [A_0 | A_1 | ...] )[M][K] @ W[K][N] )
//
// * the densenet concat of _allegro.py:278 is never materialised: A is read from up to 4
//   column segments (pointer, leading dimension, width);
// * the output is split into up to 4 column segments (latent -> [new scalars | env weights],
//   _allegro.py:284-294), each either stored or accumulated (gradient fan-in);
// * act = the MLP nonlinearity phi (NL: silu, mish or gelu) on load (second MLP layer reads the stored pre-activation);
// * epi = multiply by phi'(aux) (MLP backward, appendix B step 6).
//
// This file is the precision-generic CUDA-core path (fp64 / fp32 / bf16-storage with fp32
// accumulate): 64x64 block tile, 16-deep K slices, 4x4 register micro-tile per thread.
#include "common.cuh"

struct LinSeg {
    const void* ptr;
    int64_t ld;
    int width;
    int accum;
    const void* aux;   // A segments only: silu' multiplier source (AB2_ACT_MUL_DSILU)
    int64_t aux_ld;
};

struct LinParams {
    int64_t M;
    int K, N;
    int n_a;
    LinSeg a[AB2_MAX_SEG];
    int act;
    const void* W;
    int n_o;
    LinSeg o[AB2_MAX_SEG];
    int epi;
    const void* aux;
    int64_t aux_ld;
};

template <typename TAct, typename TAcc, int NL>
__device__ __forceinline__ TAcc lin_load_a(const LinParams& p, int64_t m, int k) {
    // locate the segment holding concat column k
#pragma unroll
    for (int s = 0; s < AB2_MAX_SEG; ++s) {
        if (s < p.n_a) {
            if (k < p.a[s].width) {
                TAcc v = to_acc<TAcc>(((const TAct*)p.a[s].ptr)[m * p.a[s].ld + k]);
                if (p.act == AB2_ACT_MUL_DSILU && p.a[s].aux)
                    v *= dact_f<NL>(to_acc<TAcc>(((const TAct*)p.a[s].aux)[m * p.a[s].aux_ld + k]));
                return v;
            }
            k -= p.a[s].width;
        }
    }
    return TAcc(0);
}

template <typename TAct, typename TAcc, int NL>
__global__ void __launch_bounds__(256) linear_kernel(const LinParams p) {
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ TAcc As[BK][BM + 4];
    __shared__ TAcc Ws[BK][BN + 4];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;
    TAcc acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = TAcc(0);

    const TAct* __restrict__ W = (const TAct*)p.W;
    for (int k0 = 0; k0 < p.K; k0 += BK) {
        // A tile: 64 rows x 16 k; consecutive threads walk k (contiguous inside a segment)
#pragma unroll
        for (int t = 0; t < (BM * BK) / 256; ++t) {
            const int e = tid + t * 256;
            const int kk = e & (BK - 1), r = e >> 4;
            const int64_t m = m0 + r;
            TAcc v = TAcc(0);
            if (m < p.M && k0 + kk < p.K) {
                v = lin_load_a<TAct, TAcc, NL>(p, m, k0 + kk);
                if (p.act == AB2_ACT_SILU) v = act_f<NL>(v);
            }
            As[kk][r] = v;
        }
#pragma unroll
        for (int t = 0; t < (BK * BN) / 256; ++t) {
            const int e = tid + t * 256;
            const int n = e & (BN - 1), kk = e >> 6;
            TAcc v = TAcc(0);
            if (k0 + kk < p.K && n0 + n < p.N) v = to_acc<TAcc>(W[(int64_t)(k0 + kk) * p.N + n0 + n]);
            Ws[kk][n] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            TAcc a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Ws[kk][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * b[j];
        }
        __syncthreads();
    }

    // epilogue
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int64_t m = m0 + ty * 4 + i;
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int n = n0 + tx * 4 + j;
            if (n >= p.N) continue;
            TAcc v = acc[i][j];
            if (p.epi == AB2_EPI_MUL_DSILU) v *= dact_f<NL>(to_acc<TAcc>(((const TAct*)p.aux)[m * p.aux_ld + n]));
#pragma unroll
            for (int s = 0; s < AB2_MAX_SEG; ++s) {
                if (s < p.n_o) {
                    if (n >= 0 && n < p.o[s].width) {
                        TAct* dst = (TAct*)p.o[s].ptr + m * p.o[s].ld + n;
                        if (p.o[s].accum) v += to_acc<TAcc>(*dst);
                        *dst = from_acc<TAct>(v);
                        n = -1 << 20;  // done
                    }
                    n -= p.o[s].width;
                }
            }
        }
    }
}

int ab2_linear_tc_try(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                      const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* Wpacked, int n_o, void* const* o_ptr, const int64_t* o_ld,
                      const int32_t* o_width, const int32_t* o_accum, int epi, const void* aux, int64_t aux_ld, cudaStream_t st, int nonlin);

extern "C" int ab2_linear_nl(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                          const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* W,
                          const void* Wpacked, int n_o, void* const* o_ptr,
                          const int64_t* o_ld, const int32_t* o_width, const int32_t* o_accum, int epi, const void* aux,
                          int64_t aux_ld, void* stream, int nonlin) {
    AB2_CHECK_ARG(nonlin == AB2_NL_SILU || nonlin == AB2_NL_MISH || nonlin == AB2_NL_GELU, "nonlinearity");
    if (M == 0) return 0;
    AB2_CHECK_ARG(n_a >= 1 && n_a <= AB2_MAX_SEG && n_o >= 1 && n_o <= AB2_MAX_SEG, "segment count");
    AB2_CHECK_ARG(K > 0 && N > 0 && W, "shape");
    AB2_CHECK_ARG(epi == AB2_EPI_NONE || aux, "aux required for dsilu epilogue");
    LinParams p;
    memset(&p, 0, sizeof(p));
    p.M = M; p.K = K; p.N = N; p.n_a = n_a; p.act = act; p.W = W; p.n_o = n_o; p.epi = epi; p.aux = aux; p.aux_ld = aux_ld;
    int ks = 0, ns = 0;
    for (int s = 0; s < n_a; ++s) {
        AB2_CHECK_ARG(a_ptr[s] && a_width[s] > 0 && a_ld[s] >= a_width[s], "A segment");
        p.a[s].ptr = a_ptr[s]; p.a[s].ld = a_ld[s]; p.a[s].width = a_width[s]; ks += a_width[s];
        p.a[s].aux = a_aux ? a_aux[s] : nullptr;
        p.a[s].aux_ld = (a_aux && a_aux_ld) ? a_aux_ld[s] : 0;
    }
    for (int s = 0; s < n_o; ++s) {
        AB2_CHECK_ARG(o_ptr[s] && o_width[s] > 0 && o_ld[s] >= o_width[s], "output segment");
        p.o[s].ptr = o_ptr[s]; p.o[s].ld = o_ld[s]; p.o[s].width = o_width[s]; p.o[s].accum = o_accum ? o_accum[s] : 0;
        ns += o_width[s];
    }
    AB2_CHECK_ARG(ks == K, "A segment widths must sum to K");
    AB2_CHECK_ARG(ns == N, "output segment widths must sum to N");
    cudaStream_t st = (cudaStream_t)stream;
    const int tc = Wpacked ? ab2_linear_tc_try(dtype, M, K, N, n_a, a_ptr, a_ld, a_width, a_aux, a_aux_ld, act, Wpacked, n_o, o_ptr, o_ld, o_width,
                                               o_accum, epi, aux, aux_ld, st, nonlin)
                           : -1;
    if (tc == 0) {
        AB2_CUDA_LAUNCH_CHECK();
        return 0;
    }
    if (tc > 0) {  // some column slices were launched, a later one could not be: the output is incomplete
        ab2_set_error("%s:%d: tensor-core linear: a column slice failed to launch (K=%d, N=%d)", __FILE__, __LINE__, K, N);
        return 2;
    }
    dim3 grid(ab2_blocks(M, 64), (unsigned)((N + 63) / 64));
    AB2_DISPATCH_NL(nonlin, AB2_DISPATCH_DTYPE(dtype, linear_kernel<TAct, TAcc, NL><<<grid, 256, 0, st>>>(p)));
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_linear(int dtype, int64_t M, int K, int N, int n_a, const void* const* a_ptr, const int64_t* a_ld,
                          const int32_t* a_width, const void* const* a_aux, const int64_t* a_aux_ld, int act, const void* W,
                          const void* Wpacked, int n_o, void* const* o_ptr,
                          const int64_t* o_ld, const int32_t* o_width, const int32_t* o_accum, int epi, const void* aux,
                          int64_t aux_ld, void* stream) {
    return ab2_linear_nl(dtype, M, K, N, n_a, a_ptr, a_ld, a_width, a_aux, a_aux_ld, act, W, Wpacked, n_o, o_ptr, o_ld, o_width, o_accum, epi, aux,
                         aux_ld, stream, AB2_NL_SILU);
}

// Harmonic force constants by central differences on local displacement clusters (phonons.force_constants).
//
// Moving atom j by h e_alpha changes only the energies of the centres C_j = {j} u {k : an edge of row k has neighbour j}
// (Allegro is strictly local), so F(r + h e) - F(r - h e) needs only the edges of the rows in C_j, each edge vector moved by
// s h e_alpha ([nbr = j] - [ctr = j]).  Four steps, all indices in the original list:
//   centres  C_j per displaced atom (count / fill), with each centre's edge offset inside the atom's cluster;
//   columns  the sorted atoms that are a centre or a neighbour of an edge of the cluster (the non-zero blocks of row j);
//   gather   a chunk of jobs (unit u = (atom a, axis alpha), sign s = +, -) as one batched CSR for the per-edge pipeline;
//   fold     -(F+ - F-) / (2h) per column from the jobs' per-edge gradients, in fp64.
// Every reduction runs in a fixed order without atomics on floating-point data, so a displaced atom's blocks do not depend
// on the chunk it ran in or on the other displaced atoms.
//
// Third-order constants (phonons.third_order_force_constants) use the same plan for pairs (j, k) of displaced atoms: the
// pairs of j are its harmonic columns, the cluster of a pair is C_j n C_k (fc3_pairs), each unit (pair, alpha, beta) is
// four jobs (fc3_gather) and the fold forms the mixed difference -(F++ - F+- - F-+ + F--) / (4h^2) (fc3_fold).
#include "common.cuh"

namespace {

constexpr int FC_THREADS = 256;
constexpr int FC_WARPS = FC_THREADS / 32;

// C_j in ascending order.  The column of j in the transposed list is in ascending edge order and edges are sorted by
// centre, so its centres arrive non-decreasing: j is merged in and repeats are skipped in one pass.
template <bool FILL>
__global__ void __launch_bounds__(FC_THREADS) fc_centres_kernel(int64_t A, const int64_t* __restrict__ atoms, const int32_t* __restrict__ col_ptr,
                                                                const int32_t* __restrict__ col_perm, const int32_t* __restrict__ ctr,
                                                                const int32_t* __restrict__ row_ptr, const int64_t* __restrict__ cptr,
                                                                int64_t* __restrict__ counts, int32_t* __restrict__ cen, int32_t* __restrict__ coff,
                                                                int64_t* __restrict__ ea) {
    const int64_t a = (int64_t)blockIdx.x * FC_THREADS + threadIdx.x;
    if (a >= A) return;
    const int32_t j = (int32_t)atoms[a];
    int64_t m = 0, off = 0;
    const int64_t base = FILL ? cptr[a] : 0;
    int32_t prev = -1;
    bool j_done = false;
    auto emit = [&](int32_t k) {
        if (FILL) {
            cen[base + m] = k;
            coff[base + m] = (int32_t)off;
            off += row_ptr[k + 1] - row_ptr[k];
        }
        ++m;
        prev = k;
    };
    for (int32_t t = col_ptr[j]; t < col_ptr[j + 1]; ++t) {
        const int32_t c = ctr[col_perm[t]];
        if (!j_done && j < c) {
            emit(j);
            j_done = true;
        }
        if (c != prev) {
            emit(c);
            if (c == j) j_done = true;
        }
    }
    if (!j_done) emit(j);
    if (FILL)
        ea[a] = off;
    else
        counts[a] = m;
}

// Columns of one displaced atom: a bitmap of the n atoms in shared memory, marked from the cluster's centres and
// neighbours (integer OR, order-free), then read out in ascending order: each thread owns a contiguous run of words, and
// an exclusive scan of the per-thread popcounts gives each run's output position.
template <bool FILL>
__global__ void __launch_bounds__(FC_THREADS) fc_columns_kernel(int64_t n, const int64_t* __restrict__ cptr, const int32_t* __restrict__ cen,
                                                                const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ nbr,
                                                                const int64_t* __restrict__ fptr, int64_t* __restrict__ counts,
                                                                int32_t* __restrict__ col) {
    extern __shared__ uint32_t bits[];
    __shared__ int64_t scan[FC_THREADS];
    const int64_t a = blockIdx.x;
    const int64_t W = (n + 31) >> 5;
    for (int64_t w = threadIdx.x; w < W; w += FC_THREADS) bits[w] = 0u;
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t c = cptr[a] + warp; c < cptr[a + 1]; c += FC_WARPS) {
        const int32_t k = cen[c];
        if (lane == 0) atomicOr(&bits[k >> 5], 1u << (k & 31));
        for (int32_t z = row_ptr[k] + lane; z < row_ptr[k + 1]; z += 32) {
            const int32_t i = nbr[z];
            atomicOr(&bits[i >> 5], 1u << (i & 31));
        }
    }
    __syncthreads();
    const int64_t per = (W + FC_THREADS - 1) / FC_THREADS;
    const int64_t w0 = threadIdx.x * per, w1 = w0 + per < W ? w0 + per : W;
    int64_t cnt = 0;
    for (int64_t w = w0; w < w1; ++w) cnt += __popc(bits[w]);
    scan[threadIdx.x] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t s = 0;
        for (int t = 0; t < FC_THREADS; ++t) {
            const int64_t v = scan[t];
            scan[t] = s;
            s += v;
        }
        if (!FILL) counts[a] = s;
    }
    __syncthreads();
    if (!FILL) return;
    int64_t o = fptr[a] + scan[threadIdx.x];
    for (int64_t w = w0; w < w1; ++w) {
        uint32_t b = bits[w];
        while (b) {
            const int bit = __ffs(b) - 1;
            col[o++] = (int32_t)(w * 32 + bit);
            b &= b - 1;
        }
    }
}

// One block per unit u = (a, alpha) of the chunk [u0, u0 + U): its two jobs (s = +1, then s = -1) side by side.  Job
// sigma of unit u starts at centre 2 (Cp[u] - Cp[u0]) + sigma m_a and edge 2 (Ep[u] - Ep[u0]) + sigma E_a.  Batched
// neighbours index past the Cb batched centres: types_b = [types[cen_b] | types] serves both ends.
template <typename TPos, typename TAcc>
__global__ void __launch_bounds__(FC_THREADS) fc_gather_kernel(int64_t u0, int64_t U, int64_t Cb, TPos h, const TPos* __restrict__ pos,
                                                               const TPos* __restrict__ shift, const int64_t* __restrict__ atoms,
                                                               const int64_t* __restrict__ cptr, const int32_t* __restrict__ cen,
                                                               const int32_t* __restrict__ coff, const int64_t* __restrict__ ea,
                                                               const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ nbr,
                                                               const int64_t* __restrict__ Cp, const int64_t* __restrict__ Ep,
                                                               int32_t* __restrict__ row_ptr_b, int32_t* __restrict__ cen_b,
                                                               int32_t* __restrict__ ctr_b, int32_t* __restrict__ nbr_b, TAcc* __restrict__ vec_b) {
    const int64_t u = u0 + blockIdx.x;
    const int64_t a = u / 3;
    const int alpha = (int)(u % 3);
    const int32_t j = (int32_t)atoms[a];
    const int64_t c0 = cptr[a], m = cptr[a + 1] - c0, Ea = ea[a];
    const int64_t cb = 2 * (Cp[u] - Cp[u0]), eb = 2 * (Ep[u] - Ep[u0]);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int sigma = 0; sigma < 2; ++sigma) {
        const TPos sh = sigma == 0 ? h : -h;
        for (int64_t c = warp; c < m; c += FC_WARPS) {
            const int32_t k = cen[c0 + c];
            const int64_t q = cb + sigma * m + c;
            const int64_t rb = eb + sigma * Ea + coff[c0 + c];
            if (lane == 0) {
                row_ptr_b[q] = (int32_t)rb;
                cen_b[q] = k;
            }
            const int32_t z0 = row_ptr[k], deg = row_ptr[k + 1] - z0;
            for (int32_t e = lane; e < deg; e += 32) {
                const int64_t z = z0 + e, zb = rb + e;
                const int32_t jn = nbr[z];
                ctr_b[zb] = (int32_t)q;
                nbr_b[zb] = (int32_t)(Cb + jn);
                const int del = (jn == j) - (k == j);
#pragma unroll
                for (int x = 0; x < 3; ++x) {
                    TPos d = pos[(int64_t)jn * 3 + x] - pos[(int64_t)k * 3 + x];
                    if (shift) d += shift[z * 3 + x];
                    if (x == alpha && del != 0) d += del > 0 ? sh : -sh;
                    vec_b[zb * 3 + x] = (TAcc)d;
                }
            }
        }
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) row_ptr_b[Cb] = (int32_t)(eb + 2 * Ea);
}

// Tangent mode (analytic force constants): one job per unit, from centre Cp[u] - Cp[u0] and edge Ep[u] - Ep[u0], the
// undisplaced edge vectors (the operations of ab2_edge_vec) and their tangent vdot_b = e_alpha ([nbr = j] - [ctr = j]).
template <typename TPos, typename TAcc>
__global__ void __launch_bounds__(FC_THREADS) fc_gather_tangent_kernel(int64_t u0, int64_t Cb, const TPos* __restrict__ pos,
                                                                       const TPos* __restrict__ shift, const int64_t* __restrict__ atoms,
                                                                       const int64_t* __restrict__ cptr, const int32_t* __restrict__ cen,
                                                                       const int32_t* __restrict__ coff, const int64_t* __restrict__ ea,
                                                                       const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ nbr,
                                                                       const int64_t* __restrict__ Cp, const int64_t* __restrict__ Ep,
                                                                       int32_t* __restrict__ row_ptr_b, int32_t* __restrict__ cen_b,
                                                                       int32_t* __restrict__ ctr_b, int32_t* __restrict__ nbr_b,
                                                                       TAcc* __restrict__ vec_b, TAcc* __restrict__ vdot_b) {
    const int64_t u = u0 + blockIdx.x;
    const int64_t a = u / 3;
    const int alpha = (int)(u % 3);
    const int32_t j = (int32_t)atoms[a];
    const int64_t c0 = cptr[a], m = cptr[a + 1] - c0;
    const int64_t cb = Cp[u] - Cp[u0], eb = Ep[u] - Ep[u0];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t c = warp; c < m; c += FC_WARPS) {
        const int32_t k = cen[c0 + c];
        const int64_t q = cb + c;
        const int64_t rb = eb + coff[c0 + c];
        if (lane == 0) {
            row_ptr_b[q] = (int32_t)rb;
            cen_b[q] = k;
        }
        const int32_t z0 = row_ptr[k], deg = row_ptr[k + 1] - z0;
        for (int32_t e = lane; e < deg; e += 32) {
            const int64_t z = z0 + e, zb = rb + e;
            const int32_t jn = nbr[z];
            ctr_b[zb] = (int32_t)q;
            nbr_b[zb] = (int32_t)(Cb + jn);
            const TAcc del = (TAcc)((jn == j) - (k == j));
#pragma unroll
            for (int x = 0; x < 3; ++x) {
                TPos d = pos[(int64_t)jn * 3 + x] - pos[(int64_t)k * 3 + x];
                if (shift) d += shift[z * 3 + x];
                vec_b[zb * 3 + x] = (TAcc)d;
                vdot_b[zb * 3 + x] = x == alpha ? del : TAcc(0);
            }
        }
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) row_ptr_b[Cb] = (int32_t)(eb + ea[a]);
}

// index of k in the ascending list s[0, m), or -1
__device__ __forceinline__ int64_t fc_find(const int32_t* __restrict__ s, int64_t m, int32_t k) {
    int64_t lo = 0, hi = m;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (s[mid] < k)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < m && s[lo] == k ? lo : -1;
}

// One block per unit u = (a, alpha), one warp per column i of row a.  F_i of a job = sum of gvec over the job's edges
// centred on i (row i, when i is in C_j) - sum over its edges with neighbour i (column i of the transposed list, kept
// when the edge's centre is in C_j).  Each lane sums (g+ - g-) in fp64 over its strided share in that order; the warp
// reduces with the fixed butterfly of warp_sum.  TANGENT: one job per unit holding the tangents of the per-edge
// gradients, folded as -F_dot (no difference, no 1/(2h): inv2h = 1).
template <typename TAcc, bool TANGENT>
__global__ void __launch_bounds__(FC_THREADS) fc_fold_kernel(int64_t u0, double inv2h, const int64_t* __restrict__ cptr,
                                                             const int32_t* __restrict__ cen, const int32_t* __restrict__ coff,
                                                             const int64_t* __restrict__ ea, const int32_t* __restrict__ row_ptr,
                                                             const int32_t* __restrict__ ctr, const int32_t* __restrict__ col_ptr,
                                                             const int32_t* __restrict__ col_perm, const int64_t* __restrict__ fptr,
                                                             const int32_t* __restrict__ col, const int64_t* __restrict__ Ep,
                                                             const TAcc* __restrict__ gvec, double* __restrict__ blocks) {
    const int64_t u = u0 + blockIdx.x;
    const int64_t a = u / 3;
    const int alpha = (int)(u % 3);
    const int64_t c0 = cptr[a], m = cptr[a + 1] - c0, Ea = ea[a];
    const int32_t* __restrict__ cs = cen + c0;
    const int64_t ep = (TANGENT ? 1 : 2) * (Ep[u] - Ep[u0]), em = ep + Ea;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int64_t p = fptr[a] + warp; p < fptr[a + 1]; p += FC_WARPS) {
        const int32_t i = col[p];
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        const int64_t ci = fc_find(cs, m, i);
        if (ci >= 0) {
            const int64_t off = coff[c0 + ci];
            const int32_t deg = row_ptr[i + 1] - row_ptr[i];
            for (int32_t e = lane; e < deg; e += 32) {
                const int64_t zp = (ep + off + e) * 3, zm = (em + off + e) * 3;
                s0 += TANGENT ? (double)gvec[zp + 0] : (double)gvec[zp + 0] - (double)gvec[zm + 0];
                s1 += TANGENT ? (double)gvec[zp + 1] : (double)gvec[zp + 1] - (double)gvec[zm + 1];
                s2 += TANGENT ? (double)gvec[zp + 2] : (double)gvec[zp + 2] - (double)gvec[zm + 2];
            }
        }
        for (int32_t t = col_ptr[i] + lane; t < col_ptr[i + 1]; t += 32) {
            const int32_t z = col_perm[t];
            const int32_t k = ctr[z];
            const int64_t ck = fc_find(cs, m, k);
            if (ck < 0) continue;
            const int64_t off = coff[c0 + ck] + (z - row_ptr[k]);
            const int64_t zp = (ep + off) * 3, zm = (em + off) * 3;
            s0 -= TANGENT ? (double)gvec[zp + 0] : (double)gvec[zp + 0] - (double)gvec[zm + 0];
            s1 -= TANGENT ? (double)gvec[zp + 1] : (double)gvec[zp + 1] - (double)gvec[zm + 1];
            s2 -= TANGENT ? (double)gvec[zp + 2] : (double)gvec[zp + 2] - (double)gvec[zm + 2];
        }
        s0 = warp_sum(s0);
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        if (lane == 0) {
            double* b = blocks + p * 9 + alpha * 3;
            b[0] = -s0 * inv2h;
            b[1] = -s1 * inv2h;
            b[2] = -s2 * inv2h;
        }
    }
}

// ---- third order (phonons.third_order_force_constants) ---------------------------------------------------------------
// A pair p = (j = pj[p], k = pk[p]) of displaced atoms changes only the energies of the centres in C_j n C_k: the 4-point
// mixed difference of any other E_c is exactly zero.  Units u = 9 p + 3 alpha + beta, each four jobs (s1, s2) = ++, +-,
// -+, -- of m_p = iptr[p+1] - iptr[p] centres and E_p = Pe[p+1] - Pe[p] edges.

// C_j n C_k by merging the two ascending lists of the all-atom centre sets (Kptr, Ken).
template <bool FILL>
__global__ void __launch_bounds__(FC_THREADS) fc3_pairs_kernel(int64_t P, const int32_t* __restrict__ pj, const int32_t* __restrict__ pk,
                                                               const int64_t* __restrict__ Kptr, const int32_t* __restrict__ Ken,
                                                               const int32_t* __restrict__ row_ptr, const int64_t* __restrict__ iptr,
                                                               int64_t* __restrict__ counts, int32_t* __restrict__ icen,
                                                               int32_t* __restrict__ ioff, int64_t* __restrict__ pe) {
    const int64_t p = (int64_t)blockIdx.x * FC_THREADS + threadIdx.x;
    if (p >= P) return;
    const int32_t j = pj[p], k = pk[p];
    int64_t x = Kptr[j], y = Kptr[k];
    const int64_t x1 = Kptr[j + 1], y1 = Kptr[k + 1];
    int64_t m = 0, off = 0;
    const int64_t base = FILL ? iptr[p] : 0;
    while (x < x1 && y < y1) {
        const int32_t a = Ken[x], b = Ken[y];
        if (a < b) {
            ++x;
        } else if (b < a) {
            ++y;
        } else {
            if (FILL) {
                icen[base + m] = a;
                ioff[base + m] = (int32_t)off;
                off += row_ptr[a + 1] - row_ptr[a];
            }
            ++m;
            ++x;
            ++y;
        }
    }
    if (FILL)
        pe[p] = off;
    else
        counts[p] = m;
}

// batched centre and edge offsets of unit u relative to the chunk start (4 jobs per unit)
__device__ __forceinline__ void fc3_unit_start(int64_t u, const int64_t* __restrict__ iptr, const int64_t* __restrict__ Pe, int64_t& c, int64_t& e) {
    const int64_t p = u / 9, r = u % 9;
    c = 9 * iptr[p] + r * (iptr[p + 1] - iptr[p]);
    e = 9 * Pe[p] + r * (Pe[p + 1] - Pe[p]);
}

// One block per unit of the chunk [u0, u0 + U): its four jobs side by side.  Job sigma starts at centre
// 4 (C(u) - C(u0)) + sigma m_p and edge 4 (E(u) - E(u0)) + sigma E_p.  delta = s1 h e_alpha ([n = j] - [c = j]) +
// s2 h e_beta ([n = k] - [c = k]) is exact (each term is 0 or +-h) and is added once, so the pair (k, j, beta, alpha)
// forms the same four edge vectors bit for bit.
template <typename TPos, typename TAcc>
__global__ void __launch_bounds__(FC_THREADS) fc3_gather_kernel(int64_t u0, int64_t Cb, TPos h, const TPos* __restrict__ pos,
                                                                const TPos* __restrict__ shift, const int32_t* __restrict__ pj,
                                                                const int32_t* __restrict__ pk, const int64_t* __restrict__ iptr,
                                                                const int32_t* __restrict__ icen, const int32_t* __restrict__ ioff,
                                                                const int64_t* __restrict__ Pe, const int32_t* __restrict__ row_ptr,
                                                                const int32_t* __restrict__ nbr, int32_t* __restrict__ row_ptr_b,
                                                                int32_t* __restrict__ cen_b, int32_t* __restrict__ ctr_b,
                                                                int32_t* __restrict__ nbr_b, TAcc* __restrict__ vec_b) {
    const int64_t u = u0 + blockIdx.x;
    const int64_t p = u / 9;
    const int alpha = (int)((u / 3) % 3), beta = (int)(u % 3);
    const int32_t j = pj[p], k = pk[p];
    const int64_t c0 = iptr[p], m = iptr[p + 1] - c0, Ep = Pe[p + 1] - Pe[p];
    int64_t cu, eu, cs, es;
    fc3_unit_start(u, iptr, Pe, cu, eu);
    fc3_unit_start(u0, iptr, Pe, cs, es);
    const int64_t cb = 4 * (cu - cs), eb = 4 * (eu - es);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int sigma = 0; sigma < 4; ++sigma) {
        const TPos s1 = sigma < 2 ? h : -h, s2 = (sigma & 1) == 0 ? h : -h;
        for (int64_t c = warp; c < m; c += FC_WARPS) {
            const int32_t kc = icen[c0 + c];
            const int64_t q = cb + sigma * m + c;
            const int64_t rb = eb + sigma * Ep + ioff[c0 + c];
            if (lane == 0) {
                row_ptr_b[q] = (int32_t)rb;
                cen_b[q] = kc;
            }
            const int32_t z0 = row_ptr[kc], deg = row_ptr[kc + 1] - z0;
            for (int32_t e = lane; e < deg; e += 32) {
                const int64_t z = z0 + e, zb = rb + e;
                const int32_t jn = nbr[z];
                ctr_b[zb] = (int32_t)q;
                nbr_b[zb] = (int32_t)(Cb + jn);
                const TPos dj = (TPos)((jn == j) - (kc == j)), dk = (TPos)((jn == k) - (kc == k));
#pragma unroll
                for (int x = 0; x < 3; ++x) {
                    TPos d = pos[(int64_t)jn * 3 + x] - pos[(int64_t)kc * 3 + x];
                    if (shift) d += shift[z * 3 + x];
                    const TPos delta = (x == alpha ? dj * s1 : (TPos)0) + (x == beta ? dk * s2 : (TPos)0);
                    d += delta;
                    vec_b[zb * 3 + x] = (TAcc)d;
                }
            }
        }
    }
    if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) row_ptr_b[Cb] = (int32_t)(eb + 4 * Ep);
}

// One block per unit, one warp per column i of pair p.  Each lane sums (g++ + g--) - (g+- + g-+) in fp64 over its
// strided share of row i (when i is in C_j n C_k) and then of column i of the transposed list (edges whose centre is in
// C_j n C_k, subtracted); the warp reduces with the fixed butterfly of warp_sum.  The pair sum is symmetric under
// swapping (j, alpha) with (k, beta), which swaps +- with -+.
template <typename TAcc>
__global__ void __launch_bounds__(FC_THREADS) fc3_fold_kernel(int64_t u0, double inv4h2, const int64_t* __restrict__ iptr,
                                                              const int32_t* __restrict__ icen, const int32_t* __restrict__ ioff,
                                                              const int64_t* __restrict__ Pe, const int32_t* __restrict__ row_ptr,
                                                              const int32_t* __restrict__ ctr, const int32_t* __restrict__ col_ptr,
                                                              const int32_t* __restrict__ col_perm, const int64_t* __restrict__ rptr,
                                                              const int32_t* __restrict__ col, const TAcc* __restrict__ gvec,
                                                              double* __restrict__ blocks) {
    const int64_t u = u0 + blockIdx.x;
    const int64_t p = u / 9;
    const int ab = (int)(u % 9);
    const int64_t c0 = iptr[p], m = iptr[p + 1] - c0, Ep = Pe[p + 1] - Pe[p];
    const int32_t* __restrict__ cs = icen + c0;
    int64_t cu, eu, cs0, es0;
    fc3_unit_start(u, iptr, Pe, cu, eu);
    fc3_unit_start(u0, iptr, Pe, cs0, es0);
    const int64_t epp = 4 * (eu - es0), epm = epp + Ep, emp = epm + Ep, emm = emp + Ep;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    auto term = [&](int64_t off, int x) {
        return ((double)gvec[(epp + off) * 3 + x] + (double)gvec[(emm + off) * 3 + x]) -
               ((double)gvec[(epm + off) * 3 + x] + (double)gvec[(emp + off) * 3 + x]);
    };
    for (int64_t t = rptr[p] + warp; t < rptr[p + 1]; t += FC_WARPS) {
        const int32_t i = col[t];
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        const int64_t ci = fc_find(cs, m, i);
        if (ci >= 0) {
            const int64_t off = ioff[c0 + ci];
            const int32_t deg = row_ptr[i + 1] - row_ptr[i];
            for (int32_t e = lane; e < deg; e += 32) {
                s0 += term(off + e, 0);
                s1 += term(off + e, 1);
                s2 += term(off + e, 2);
            }
        }
        for (int32_t w = col_ptr[i] + lane; w < col_ptr[i + 1]; w += 32) {
            const int32_t z = col_perm[w];
            const int32_t kc = ctr[z];
            const int64_t ck = fc_find(cs, m, kc);
            if (ck < 0) continue;
            const int64_t off = ioff[c0 + ck] + (z - row_ptr[kc]);
            s0 -= term(off, 0);
            s1 -= term(off, 1);
            s2 -= term(off, 2);
        }
        s0 = warp_sum(s0);
        s1 = warp_sum(s1);
        s2 = warp_sum(s2);
        if (lane == 0) {
            double* b = blocks + t * 27 + ab * 3;
            b[0] = -s0 * inv4h2;
            b[1] = -s1 * inv4h2;
            b[2] = -s2 * inv4h2;
        }
    }
}

}  // namespace

extern "C" int ab2_fc_centres_count(int64_t A, const int64_t* atoms, const int32_t* col_ptr, const int32_t* col_perm, const int32_t* ctr,
                                    int64_t* counts, void* stream) {
    AB2_CHECK_ARG(A >= 0, "sizes");
    if (A == 0) return 0;
    AB2_CHECK_ARG(atoms && col_ptr && ctr && counts, "null pointer");
    fc_centres_kernel<false><<<ab2_blocks(A, FC_THREADS), FC_THREADS, 0, (cudaStream_t)stream>>>(A, atoms, col_ptr, col_perm, ctr, nullptr,
                                                                                                 nullptr, counts, nullptr, nullptr, nullptr);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc_centres_fill(int64_t A, const int64_t* atoms, const int32_t* col_ptr, const int32_t* col_perm, const int32_t* ctr,
                                   const int32_t* row_ptr, const int64_t* cptr, int32_t* cen, int32_t* coff, int64_t* ea, void* stream) {
    AB2_CHECK_ARG(A >= 0, "sizes");
    if (A == 0) return 0;
    AB2_CHECK_ARG(atoms && col_ptr && ctr && row_ptr && cptr && cen && coff && ea, "null pointer");
    fc_centres_kernel<true><<<ab2_blocks(A, FC_THREADS), FC_THREADS, 0, (cudaStream_t)stream>>>(A, atoms, col_ptr, col_perm, ctr, row_ptr,
                                                                                                cptr, nullptr, cen, coff, ea);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc_columns(int fill, int64_t A, int64_t n, const int64_t* cptr, const int32_t* cen, const int32_t* row_ptr,
                              const int32_t* nbr, const int64_t* fptr, int64_t* counts, int32_t* col, void* stream) {
    AB2_CHECK_ARG(A >= 0 && n >= 1 && n <= AB2_FC_MAX_ATOMS, "atoms: 1 .. AB2_FC_MAX_ATOMS");
    AB2_CHECK_ARG(A <= 0x7fffffffLL, "too many displaced atoms for one launch");
    if (A == 0) return 0;
    AB2_CHECK_ARG(cptr && cen && row_ptr && (fill ? (fptr && col) : counts != nullptr), "null pointer");
    const size_t smem = (size_t)((n + 31) >> 5) * sizeof(uint32_t);
    cudaStream_t st = (cudaStream_t)stream;
    if (fill) {
        AB2_CUDA_CALL(cudaFuncSetAttribute(fc_columns_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        fc_columns_kernel<true><<<(unsigned)A, FC_THREADS, smem, st>>>(n, cptr, cen, row_ptr, nbr, fptr, nullptr, col);
    } else {
        AB2_CUDA_CALL(cudaFuncSetAttribute(fc_columns_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        fc_columns_kernel<false><<<(unsigned)A, FC_THREADS, smem, st>>>(n, cptr, cen, row_ptr, nbr, nullptr, counts, nullptr);
    }
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc_gather(int pos_dtype, int acc_dtype, int64_t u0, int64_t U, int64_t Cb, double h, const void* pos, const void* shift,
                             const int64_t* atoms, const int64_t* cptr, const int32_t* cen, const int32_t* coff, const int64_t* ea,
                             const int32_t* row_ptr, const int32_t* nbr, const int64_t* Cp, const int64_t* Ep, int32_t* row_ptr_b,
                             int32_t* cen_b, int32_t* ctr_b, int32_t* nbr_b, void* vec_b, void* stream) {
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "edge vectors must be fp64 or fp32");
    AB2_CHECK_ARG(u0 >= 0 && U >= 1 && U <= 0x7fffffffLL && Cb >= 1 && Cb <= 0x7fffffffLL, "sizes");
    AB2_CHECK_ARG(pos && atoms && cptr && cen && coff && ea && row_ptr && Cp && Ep && row_ptr_b && cen_b, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned g = (unsigned)U;
#define AB2_FC_GATHER(TP, TA)                                                                                                   \
    fc_gather_kernel<TP, TA><<<g, FC_THREADS, 0, st>>>(u0, U, Cb, (TP)h, (const TP*)pos, (const TP*)shift, atoms, cptr, cen, coff, ea, \
                                                       row_ptr, nbr, Cp, Ep, row_ptr_b, cen_b, ctr_b, nbr_b, (TA*)vec_b)
    if (pos_dtype == AB2_F64 && acc_dtype == AB2_F64)
        AB2_FC_GATHER(double, double);
    else if (pos_dtype == AB2_F64)
        AB2_FC_GATHER(double, float);
    else if (acc_dtype == AB2_F64)
        AB2_FC_GATHER(float, double);
    else
        AB2_FC_GATHER(float, float);
#undef AB2_FC_GATHER
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc_fold(int acc_dtype, int64_t u0, int64_t U, double h, const int64_t* cptr, const int32_t* cen, const int32_t* coff,
                           const int64_t* ea, const int32_t* row_ptr, const int32_t* ctr, const int32_t* col_ptr, const int32_t* col_perm,
                           const int64_t* fptr, const int32_t* col, const int64_t* Ep, const void* gvec, double* blocks, void* stream) {
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "gradients must be fp64 or fp32");
    AB2_CHECK_ARG(u0 >= 0 && U >= 1 && U <= 0x7fffffffLL, "sizes");
    AB2_CHECK_ARG(h > 0.0, "displacement must be > 0");
    AB2_CHECK_ARG(cptr && cen && coff && ea && row_ptr && col_ptr && fptr && col && Ep && blocks, "null pointer");
    const double inv2h = 1.0 / (2.0 * h);
    cudaStream_t st = (cudaStream_t)stream;
    if (acc_dtype == AB2_F64)
        fc_fold_kernel<double, false><<<(unsigned)U, FC_THREADS, 0, st>>>(u0, inv2h, cptr, cen, coff, ea, row_ptr, ctr, col_ptr, col_perm, fptr, col, Ep,
                                                                   (const double*)gvec, blocks);
    else
        fc_fold_kernel<float, false><<<(unsigned)U, FC_THREADS, 0, st>>>(u0, inv2h, cptr, cen, coff, ea, row_ptr, ctr, col_ptr, col_perm, fptr, col, Ep,
                                                                  (const float*)gvec, blocks);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc_gather_tangent(int pos_dtype, int acc_dtype, int64_t u0, int64_t U, int64_t Cb, const void* pos, const void* shift,
                                     const int64_t* atoms, const int64_t* cptr, const int32_t* cen, const int32_t* coff, const int64_t* ea,
                                     const int32_t* row_ptr, const int32_t* nbr, const int64_t* Cp, const int64_t* Ep, int32_t* row_ptr_b,
                                     int32_t* cen_b, int32_t* ctr_b, int32_t* nbr_b, void* vec_b, void* vdot_b, void* stream) {
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "edge vectors must be fp64 or fp32");
    AB2_CHECK_ARG(u0 >= 0 && U >= 1 && U <= 0x7fffffffLL && Cb >= 1 && Cb <= 0x7fffffffLL, "sizes");
    AB2_CHECK_ARG(pos && atoms && cptr && cen && coff && ea && row_ptr && Cp && Ep && row_ptr_b && cen_b, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned g = (unsigned)U;
#define AB2_FC_GATHER_T(TP, TA)                                                                                                       \
    fc_gather_tangent_kernel<TP, TA><<<g, FC_THREADS, 0, st>>>(u0, Cb, (const TP*)pos, (const TP*)shift, atoms, cptr, cen, coff, ea, row_ptr, \
                                                               nbr, Cp, Ep, row_ptr_b, cen_b, ctr_b, nbr_b, (TA*)vec_b, (TA*)vdot_b)
    if (pos_dtype == AB2_F64 && acc_dtype == AB2_F64)
        AB2_FC_GATHER_T(double, double);
    else if (pos_dtype == AB2_F64)
        AB2_FC_GATHER_T(double, float);
    else if (acc_dtype == AB2_F64)
        AB2_FC_GATHER_T(float, double);
    else
        AB2_FC_GATHER_T(float, float);
#undef AB2_FC_GATHER_T
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc_fold_tangent(int acc_dtype, int64_t u0, int64_t U, const int64_t* cptr, const int32_t* cen, const int32_t* coff,
                                   const int64_t* ea, const int32_t* row_ptr, const int32_t* ctr, const int32_t* col_ptr, const int32_t* col_perm,
                                   const int64_t* fptr, const int32_t* col, const int64_t* Ep, const void* gvec_dot, double* blocks, void* stream) {
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "gradients must be fp64 or fp32");
    AB2_CHECK_ARG(u0 >= 0 && U >= 1 && U <= 0x7fffffffLL, "sizes");
    AB2_CHECK_ARG(cptr && cen && coff && ea && row_ptr && col_ptr && fptr && col && Ep && blocks, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (acc_dtype == AB2_F64)
        fc_fold_kernel<double, true><<<(unsigned)U, FC_THREADS, 0, st>>>(u0, 1.0, cptr, cen, coff, ea, row_ptr, ctr, col_ptr, col_perm, fptr, col, Ep,
                                                                         (const double*)gvec_dot, blocks);
    else
        fc_fold_kernel<float, true><<<(unsigned)U, FC_THREADS, 0, st>>>(u0, 1.0, cptr, cen, coff, ea, row_ptr, ctr, col_ptr, col_perm, fptr, col, Ep,
                                                                        (const float*)gvec_dot, blocks);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc3_pairs_count(int64_t P, const int32_t* pj, const int32_t* pk, const int64_t* Kptr, const int32_t* Ken, int64_t* counts,
                                   void* stream) {
    AB2_CHECK_ARG(P >= 0, "sizes");
    if (P == 0) return 0;
    AB2_CHECK_ARG(pj && pk && Kptr && Ken && counts, "null pointer");
    fc3_pairs_kernel<false><<<ab2_blocks(P, FC_THREADS), FC_THREADS, 0, (cudaStream_t)stream>>>(P, pj, pk, Kptr, Ken, nullptr, nullptr, counts,
                                                                                                nullptr, nullptr, nullptr);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc3_pairs_fill(int64_t P, const int32_t* pj, const int32_t* pk, const int64_t* Kptr, const int32_t* Ken, const int32_t* row_ptr,
                                  const int64_t* iptr, int32_t* icen, int32_t* ioff, int64_t* pe, void* stream) {
    AB2_CHECK_ARG(P >= 0, "sizes");
    if (P == 0) return 0;
    AB2_CHECK_ARG(pj && pk && Kptr && Ken && row_ptr && iptr && icen && ioff && pe, "null pointer");
    fc3_pairs_kernel<true><<<ab2_blocks(P, FC_THREADS), FC_THREADS, 0, (cudaStream_t)stream>>>(P, pj, pk, Kptr, Ken, row_ptr, iptr, nullptr, icen,
                                                                                               ioff, pe);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc3_gather(int pos_dtype, int acc_dtype, int64_t u0, int64_t U, int64_t Cb, double h, const void* pos, const void* shift,
                              const int32_t* pj, const int32_t* pk, const int64_t* iptr, const int32_t* icen, const int32_t* ioff,
                              const int64_t* Pe, const int32_t* row_ptr, const int32_t* nbr, int32_t* row_ptr_b, int32_t* cen_b,
                              int32_t* ctr_b, int32_t* nbr_b, void* vec_b, void* stream) {
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "edge vectors must be fp64 or fp32");
    AB2_CHECK_ARG(u0 >= 0 && U >= 1 && U <= 0x7fffffffLL && Cb >= 1 && Cb <= 0x7fffffffLL, "sizes");
    AB2_CHECK_ARG(pos && pj && pk && iptr && icen && ioff && Pe && row_ptr && nbr && row_ptr_b && cen_b && ctr_b && nbr_b && vec_b,
                  "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned g = (unsigned)U;
#define AB2_FC3_GATHER(TP, TA)                                                                                                         \
    fc3_gather_kernel<TP, TA><<<g, FC_THREADS, 0, st>>>(u0, Cb, (TP)h, (const TP*)pos, (const TP*)shift, pj, pk, iptr, icen, ioff, Pe, \
                                                        row_ptr, nbr, row_ptr_b, cen_b, ctr_b, nbr_b, (TA*)vec_b)
    if (pos_dtype == AB2_F64 && acc_dtype == AB2_F64)
        AB2_FC3_GATHER(double, double);
    else if (pos_dtype == AB2_F64)
        AB2_FC3_GATHER(double, float);
    else if (acc_dtype == AB2_F64)
        AB2_FC3_GATHER(float, double);
    else
        AB2_FC3_GATHER(float, float);
#undef AB2_FC3_GATHER
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_fc3_fold(int acc_dtype, int64_t u0, int64_t U, double h, const int64_t* iptr, const int32_t* icen, const int32_t* ioff,
                            const int64_t* Pe, const int32_t* row_ptr, const int32_t* ctr, const int32_t* col_ptr, const int32_t* col_perm,
                            const int64_t* rptr, const int32_t* col, const void* gvec, double* blocks, void* stream) {
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "gradients must be fp64 or fp32");
    AB2_CHECK_ARG(u0 >= 0 && U >= 1 && U <= 0x7fffffffLL, "sizes");
    AB2_CHECK_ARG(h > 0.0, "displacement must be > 0");
    AB2_CHECK_ARG(iptr && icen && ioff && Pe && row_ptr && col_ptr && rptr && col && blocks, "null pointer");
    const double inv4h2 = 1.0 / (4.0 * h * h);
    cudaStream_t st = (cudaStream_t)stream;
    if (acc_dtype == AB2_F64)
        fc3_fold_kernel<double><<<(unsigned)U, FC_THREADS, 0, st>>>(u0, inv4h2, iptr, icen, ioff, Pe, row_ptr, ctr, col_ptr, col_perm, rptr, col,
                                                                    (const double*)gvec, blocks);
    else
        fc3_fold_kernel<float><<<(unsigned)U, FC_THREADS, 0, st>>>(u0, inv4h2, iptr, icen, ioff, Pe, row_ptr, ctr, col_ptr, col_perm, rptr, col,
                                                                   (const float*)gvec, blocks);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

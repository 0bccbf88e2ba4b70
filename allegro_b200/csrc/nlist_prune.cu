// Per-edge-type pruning of a centre-sorted neighbour list: keep edge z (centre i, neighbour j, shift s) iff
//   d2 < cut2[t_i * T + t_j],   d2 = sum_x (pos[j][x] + s[x] - pos[i][x])^2
// with d2 in fp64 from the stored positions and shifts (fp32 values convert exactly) by explicit _rn operations in a
// fixed order (x, y, z), so that a torch restatement matches it bit for bit.  cut2 is the [T, T] fp64 table of squared
// list radii, DIRECTED (row = centre type), as the model's rmax_table is indexed.
//
// One pass over any list source (the cell lists, the batched-frames search, the slab lists): an edge beyond its pair's
// cutoff contributes an exact zero to every output of the model (x = r / r_ab >= 1 zeroes the radial basis, the spline
// basis and the ZBL cutoff, and every MLP is bias-free), so the step is cheaper by the edges removed.
//   prune_count : one warp per centre row, lanes over the row in chunks of 32, kept edges counted with ballot + popc
//   prune_fill  : the same predicate, kept edges written in row order at out_row_ptr[i] + (kept lanes below)
// Between them the host takes the prefix sum of the counts.  The pruned row is an ordered subsequence of the input row;
// nbr and the shift are copied bitwise.
#include "common.cuh"

namespace {

constexpr int PRUNE_WARPS = 8;  // rows per 256-thread block

// fp64 squared length of edge z, in the order the header documents
template <typename T>
__device__ __forceinline__ double prune_d2(const T* __restrict__ pos, int64_t i, int64_t j, const T* __restrict__ shift, int64_t z) {
    double d2 = 0.0;
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        const double d = __dsub_rn(__dadd_rn((double)pos[j * 3 + x], (double)shift[z * 3 + x]), (double)pos[i * 3 + x]);
        d2 = x == 0 ? __dmul_rn(d, d) : __dadd_rn(d2, __dmul_rn(d, d));
    }
    return d2;
}

// FILL = false: counts[i] = kept edges of row i; FILL = true: kept nbr / shift rows from out_row_ptr[i]
template <typename T, bool FILL>
__global__ void __launch_bounds__(PRUNE_WARPS * 32) prune_kernel(int64_t n_centres, int num_types, const T* __restrict__ pos,
                                                                const int32_t* __restrict__ types, const double* __restrict__ cut2,
                                                                const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ nbr,
                                                                const T* __restrict__ shift, int32_t* __restrict__ counts,
                                                                const int32_t* __restrict__ out_row_ptr, int32_t* __restrict__ out_nbr,
                                                                T* __restrict__ out_shift) {
    const int64_t i = (int64_t)blockIdx.x * PRUNE_WARPS + (threadIdx.x >> 5);
    if (i >= n_centres) return;  // whole warps leave together: the ballots below see full warps
    const int lane = threadIdx.x & 31;
    const int e0 = row_ptr[i], e1 = row_ptr[i + 1];
    const double* __restrict__ crow = cut2 + (int64_t)types[i] * num_types;
    int out = FILL ? out_row_ptr[i] : 0;
    for (int c = e0; c < e1; c += 32) {
        const int z = c + lane;
        bool keep = false;
        int32_t j = 0;
        if (z < e1) {
            j = nbr[z];
            keep = prune_d2(pos, i, (int64_t)j, shift, z) < crow[types[j]];
        }
        const unsigned mask = __ballot_sync(0xffffffffu, keep);
        if (FILL && keep) {
            const int o = out + __popc(mask & ((1u << lane) - 1u));
            out_nbr[o] = j;
#pragma unroll
            for (int x = 0; x < 3; ++x) out_shift[(int64_t)o * 3 + x] = shift[(int64_t)z * 3 + x];
        }
        out += __popc(mask);
    }
    if (!FILL && lane == 0) counts[i] = out;
}

}  // namespace

extern "C" int ab2_nl_prune_count(int pos_dtype, int64_t n_centres, int64_t n_edges, int num_types, const void* pos, const int32_t* types,
                                  const double* cut2, const int32_t* row_ptr, const int32_t* nbr, const void* shift, int32_t* counts,
                                  void* stream) {
    AB2_CHECK_ARG(n_centres >= 0 && n_edges >= 0 && n_edges < (int64_t)0x7fffffff, "sizes (0 <= edges < 2^31 - 1)");
    AB2_CHECK_ARG(num_types >= 1, "num_types >= 1");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    if (n_centres == 0 || n_edges == 0) return 0;
    AB2_CHECK_ARG(pos && types && cut2 && row_ptr && nbr && shift && counts, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = ab2_blocks(n_centres, PRUNE_WARPS);
    if (pos_dtype == AB2_F64)
        prune_kernel<double, false><<<blocks, PRUNE_WARPS * 32, 0, st>>>(n_centres, num_types, (const double*)pos, types, cut2, row_ptr, nbr,
                                                                         (const double*)shift, counts, nullptr, nullptr, nullptr);
    else
        prune_kernel<float, false><<<blocks, PRUNE_WARPS * 32, 0, st>>>(n_centres, num_types, (const float*)pos, types, cut2, row_ptr, nbr,
                                                                        (const float*)shift, counts, nullptr, nullptr, nullptr);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_nl_prune_fill(int pos_dtype, int64_t n_centres, int64_t n_edges, int num_types, const void* pos, const int32_t* types,
                                 const double* cut2, const int32_t* row_ptr, const int32_t* nbr, const void* shift,
                                 const int32_t* out_row_ptr, int32_t* out_nbr, void* out_shift, void* stream) {
    AB2_CHECK_ARG(n_centres >= 0 && n_edges >= 0 && n_edges < (int64_t)0x7fffffff, "sizes (0 <= edges < 2^31 - 1)");
    AB2_CHECK_ARG(num_types >= 1, "num_types >= 1");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    if (n_centres == 0 || n_edges == 0) return 0;
    AB2_CHECK_ARG(pos && types && cut2 && row_ptr && nbr && shift && out_row_ptr && out_nbr && out_shift, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = ab2_blocks(n_centres, PRUNE_WARPS);
    if (pos_dtype == AB2_F64)
        prune_kernel<double, true><<<blocks, PRUNE_WARPS * 32, 0, st>>>(n_centres, num_types, (const double*)pos, types, cut2, row_ptr, nbr,
                                                                        (const double*)shift, nullptr, out_row_ptr, out_nbr, (double*)out_shift);
    else
        prune_kernel<float, true><<<blocks, PRUNE_WARPS * 32, 0, st>>>(n_centres, num_types, (const float*)pos, types, cut2, row_ptr, nbr,
                                                                       (const float*)shift, nullptr, out_row_ptr, out_nbr, (float*)out_shift);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

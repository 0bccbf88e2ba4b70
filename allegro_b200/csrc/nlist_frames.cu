// All-pairs neighbour search for a batch of small frames, emitted in the centre-sorted CSR format every kernel consumes.
//
// The cell list of nlist.cu needs an orthorhombic box at least 3 r_max wide on every periodic axis.  Small cells (a
// 64-atom Si cell is 2.7 r_max at r_max 4), triclinic cells and molecules fall outside it.  These kernels take any cell
// the torch all-pairs search of data.neighbor_list accepts, for thousands of frames in one launch:
//   nlf_walk<COUNT> : number of neighbours of every centre
//   nlf_walk<FILL>  : the same walk writing nbr[row_ptr[i] + k] and the shift VECTOR of each edge
// The walk itself (one warp per centre, rows ordered by neighbour, then image) is in nlist_frames.cuh.
#include "nlist_frames.cuh"

namespace {

template <bool FILL>
int nlf_launch(int pos_dtype, int64_t n, int64_t B, const int32_t* frame_ptr, const void* pos, const void* cell, const void* inv,
               const int32_t* pbc, const int32_t* nimg, double r_max, int32_t* counts, const int32_t* row_ptr, int32_t* nbr, void* shift,
               void* stream) {
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    AB2_CHECK_ARG(B >= 1 && frame_ptr && pos && cell && inv && pbc && nimg, "null pointer or no frame");
    AB2_CHECK_ARG(r_max > 0, "r_max must be positive");
    AB2_CHECK_ARG(FILL ? (row_ptr && nbr && shift) : (counts != nullptr), "null output pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = ab2_blocks(n, NLF_WARPS);
    if (pos_dtype == AB2_F64)
        nlf_walk_kernel<double, FILL><<<grid, NLF_WARPS * 32, 0, st>>>(n, B, frame_ptr, (const double*)pos, (const double*)cell,
                                                                      (const double*)inv, pbc, nimg, r_max, counts, row_ptr, nbr, (double*)shift);
    else
        nlf_walk_kernel<float, FILL><<<grid, NLF_WARPS * 32, 0, st>>>(n, B, frame_ptr, (const float*)pos, (const float*)cell,
                                                                     (const float*)inv, pbc, nimg, r_max, counts, row_ptr, nbr, (float*)shift);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int ab2_nl_frames_count(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos,
                                   const void* cell, const void* inv_cell, const int32_t* pbc, const int32_t* nimg, double r_max,
                                   int32_t* counts, void* stream) {
    return nlf_launch<false>(pos_dtype, n, n_frames, frame_ptr, pos, cell, inv_cell, pbc, nimg, r_max, counts, nullptr, nullptr, nullptr,
                             stream);
}

extern "C" int ab2_nl_frames_fill(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos,
                                  const void* cell, const void* inv_cell, const int32_t* pbc, const int32_t* nimg, double r_max,
                                  const int32_t* row_ptr, int32_t* nbr, void* shift, void* stream) {
    return nlf_launch<true>(pos_dtype, n, n_frames, frame_ptr, pos, cell, inv_cell, pbc, nimg, r_max, nullptr, row_ptr, nbr, shift, stream);
}

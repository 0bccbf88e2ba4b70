// Cell-list neighbour search on the device, emitted directly in the centre-sorted CSR format every kernel
// consumes (SURVEY section 8 row f2: "GPU neighbour list + centre sort").
//
// The reference takes `edge_index` [2,E] int64 from nequip's data pipeline / LAMMPS (allegro/nn/_allegro.py:238,
// allegro/_compile.py:41-61); building 5x10^7 int64 pairs with torch ops and sorting them by centre costs more
// memory traffic than the model evaluation itself at the 1M-atom scale.  Here: orthorhombic box, per-axis
// periodicity, cells of edge >= r_max (>= 3 cells on every periodic axis), three small kernels:
//   nl_bin   : wrapped position, image offset of the raw position, cell id      (one thread per atom)
//   nl_count : neighbours within r_max of every CENTRE (owned atoms come first)  (one thread per centre, 27 cells)
//   nl_fill  : the same walk writing nbr[row_ptr[i] + k] and the shift VECTOR of each edge
// Between them the host sorts atoms by cell id and takes two prefix sums (plumbing).  Rows come out in cell-walk
// order, which is fixed for a given frame: the summation order of every segmented reduction is reproducible.
//   r = pos[nbr] + shift - pos[ctr]   holds for the RAW (unwrapped) positions.
#include "common.cuh"

namespace {

struct NlGeom {
    double box[3], origin[3];
    int pbc[3], ncell[3];
    double rmax2;
};

template <typename T>
__device__ __forceinline__ void nl_wrap(const NlGeom& g, const T* __restrict__ pos, int64_t i, T (&w)[3], int (&img)[3], int (&c)[3]) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const T rel = pos[i * 3 + a] - (T)g.origin[a];
        const T L = (T)g.box[a];
        img[a] = g.pbc[a] ? (int)floor(rel / L) : 0;
        w[a] = rel - (T)img[a] * L;
        int ci = (int)(w[a] / L * (T)g.ncell[a]);
        c[a] = ci < 0 ? 0 : (ci >= g.ncell[a] ? g.ncell[a] - 1 : ci);
    }
}

template <typename T>
__global__ void __launch_bounds__(256) nl_bin_kernel(NlGeom g, int64_t n, const T* __restrict__ pos, int32_t* __restrict__ cell_id) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    T w[3];
    int img[3], c[3];
    nl_wrap(g, pos, i, w, img, c);
    cell_id[i] = (c[0] * g.ncell[1] + c[1]) * g.ncell[2] + c[2];
}

// FILL = false: counts[i]; FILL = true: nbr / shift rows at row_ptr[i]
template <typename T, bool FILL>
__global__ void __launch_bounds__(128) nl_walk_kernel(NlGeom g, int64_t n_centres, const T* __restrict__ pos,
                                                      const int32_t* __restrict__ cell_start, const int32_t* __restrict__ order,
                                                      int32_t* __restrict__ counts, const int32_t* __restrict__ row_ptr,
                                                      int32_t* __restrict__ nbr, T* __restrict__ shift) {
    const int64_t i = (int64_t)blockIdx.x * 128 + threadIdx.x;
    if (i >= n_centres) return;
    T wi[3];
    int imgi[3], ci[3];
    nl_wrap(g, pos, i, wi, imgi, ci);
    int cnt = 0;
    int64_t out = FILL ? row_ptr[i] : 0;
    for (int dx = -1; dx <= 1; ++dx)
        for (int dy = -1; dy <= 1; ++dy)
            for (int dz = -1; dz <= 1; ++dz) {
                const int d[3] = {dx, dy, dz};
                int cw[3], im[3];
                bool ok = true;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const int c = ci[a] + d[a];
                    im[a] = c < 0 ? -1 : (c >= g.ncell[a] ? 1 : 0);
                    if (im[a] != 0 && !g.pbc[a]) ok = false;
                    cw[a] = c - im[a] * g.ncell[a];
                }
                if (!ok) continue;
                const int cell = (cw[0] * g.ncell[1] + cw[1]) * g.ncell[2] + cw[2];
                const int a0 = cell_start[cell], a1 = cell_start[cell + 1];
                for (int a = a0; a < a1; ++a) {
                    const int64_t j = order[a];
                    T wj[3];
                    int imgj[3], cj[3];
                    nl_wrap(g, pos, j, wj, imgj, cj);
                    T r2 = 0;
                    T sh[3];
#pragma unroll
                    for (int x = 0; x < 3; ++x) {
                        const T rx = wj[x] + (T)im[x] * (T)g.box[x] - wi[x];
                        r2 += rx * rx;
                        sh[x] = (T)(im[x] - imgj[x] + imgi[x]) * (T)g.box[x];
                    }
                    if (r2 < (T)g.rmax2 && !(j == i && im[0] == 0 && im[1] == 0 && im[2] == 0)) {
                        if (FILL) {
                            nbr[out] = (int32_t)j;
                            shift[out * 3 + 0] = sh[0];
                            shift[out * 3 + 1] = sh[1];
                            shift[out * 3 + 2] = sh[2];
                            ++out;
                        }
                        ++cnt;
                    }
                }
            }
    if (!FILL) counts[i] = cnt;
}

int nl_geom(NlGeom& g, const double* box, const double* origin, const int32_t* pbc, const int32_t* ncell, double r_max) {
    for (int a = 0; a < 3; ++a) {
        g.box[a] = box[a]; g.origin[a] = origin[a]; g.pbc[a] = pbc[a]; g.ncell[a] = ncell[a];
        if (!(box[a] > 0) || ncell[a] < 1) return 1;
        if (pbc[a] && ncell[a] < 3) return 2;                 // a periodic axis would visit the same cell twice
        if (box[a] / ncell[a] < r_max * (1 - 1e-12)) return 3;  // cells must be at least r_max wide
    }
    // cell ids and cell_start offsets are int32 (a far-flung atom on an open axis asks for billions of cells: the host
    // coarsens such grids, data.cell_grid)
    if ((int64_t)ncell[0] * ncell[1] * ncell[2] >= (int64_t)0x7fffffff) return 4;
    g.rmax2 = r_max * r_max;
    return 0;
}

}  // namespace

extern "C" int ab2_nl_bin(int pos_dtype, int64_t n, const void* pos, const double* box_host, const double* origin_host,
                          const int32_t* pbc_host, const int32_t* ncell_host, double r_max, int32_t* cell_id, void* stream) {
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos && cell_id && box_host && origin_host && pbc_host && ncell_host, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    NlGeom g;
    AB2_CHECK_ARG(nl_geom(g, box_host, origin_host, pbc_host, ncell_host, r_max) == 0, "box / cell grid (need cells >= r_max, >= 3 cells per periodic axis, < 2^31 cells)");
    cudaStream_t st = (cudaStream_t)stream;
    if (pos_dtype == AB2_F64) nl_bin_kernel<double><<<ab2_blocks(n, 256), 256, 0, st>>>(g, n, (const double*)pos, cell_id);
    else nl_bin_kernel<float><<<ab2_blocks(n, 256), 256, 0, st>>>(g, n, (const float*)pos, cell_id);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_nl_count(int pos_dtype, int64_t n_centres, const void* pos, const double* box_host, const double* origin_host,
                            const int32_t* pbc_host, const int32_t* ncell_host, double r_max, const int32_t* cell_start,
                            const int32_t* order, int32_t* counts, void* stream) {
    if (n_centres == 0) return 0;
    AB2_CHECK_ARG(pos && cell_start && order && counts, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    NlGeom g;
    AB2_CHECK_ARG(nl_geom(g, box_host, origin_host, pbc_host, ncell_host, r_max) == 0, "box / cell grid");
    cudaStream_t st = (cudaStream_t)stream;
    if (pos_dtype == AB2_F64)
        nl_walk_kernel<double, false><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const double*)pos, cell_start, order, counts, nullptr, nullptr, nullptr);
    else
        nl_walk_kernel<float, false><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const float*)pos, cell_start, order, counts, nullptr, nullptr, nullptr);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_nl_fill(int pos_dtype, int64_t n_centres, const void* pos, const double* box_host, const double* origin_host,
                           const int32_t* pbc_host, const int32_t* ncell_host, double r_max, const int32_t* cell_start,
                           const int32_t* order, const int32_t* row_ptr, int32_t* nbr, void* shift, void* stream) {
    if (n_centres == 0) return 0;
    AB2_CHECK_ARG(pos && cell_start && order && row_ptr && nbr && shift, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    NlGeom g;
    AB2_CHECK_ARG(nl_geom(g, box_host, origin_host, pbc_host, ncell_host, r_max) == 0, "box / cell grid");
    cudaStream_t st = (cudaStream_t)stream;
    if (pos_dtype == AB2_F64)
        nl_walk_kernel<double, true><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const double*)pos, cell_start, order, nullptr, row_ptr, nbr, (double*)shift);
    else
        nl_walk_kernel<float, true><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const float*)pos, cell_start, order, nullptr, row_ptr, nbr, (float*)shift);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

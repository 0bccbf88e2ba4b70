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
//
// The LATTICE instantiations (ab2_nl_lattice_*) take any non-singular cell: atoms are binned in fractional
// coordinates f = pos . h^-1 - origin (h = the rows a, b, c), bins are parallelepipeds of thickness t_a = H_a / n_a
// (H_a = |det h| / |h_p x h_q|, the height of the cell along a), and each centre walks k_a = ceil(r_max / t_a) bins
// either side on every axis.  Distinct offsets are distinct (bin, image) pairs, so a periodic axis of 1 or 2 bins, or
// one shorter than r_max (k_a > 1), needs no extra rule and yields no duplicate row.  Wrap, bin and distance test run
// in fp64 for both position dtypes (an fp32 frame gets the fp64 pair set of its fp32 positions); the shift
// (im - img0[j] + img0[i]) . h is rounded once to the positions' dtype.
#include <cmath>
#include <type_traits>

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

// general lattice: binning rows h[a][x] (row a = lattice vector a), hinv = h^-1 (f = pos . hinv - origin), fractional
// origin, k_a = reach[a] bins walked either side of the centre's bin on axis a
struct NlLatticeGeom {
    double h[3][3], hinv[3][3], origin[3];
    int pbc[3], ncell[3], reach[3];
    double rmax2;
};

template <bool LATTICE>
using NlGeomOf = std::conditional_t<LATTICE, NlLatticeGeom, NlGeom>;

// wrapped position (fp64), image of the raw position along the periodic axes, bin
template <typename T>
__device__ __forceinline__ void nl_lattice_wrap(const NlLatticeGeom& g, const T* __restrict__ pos, int64_t i, double (&w)[3], int (&img)[3],
                                                int (&c)[3]) {
    const double p[3] = {(double)pos[i * 3 + 0], (double)pos[i * 3 + 1], (double)pos[i * 3 + 2]};
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double f = p[0] * g.hinv[0][a] + p[1] * g.hinv[1][a] + p[2] * g.hinv[2][a] - g.origin[a];
        // the conversions saturate (and take NaN to 0): an exploded frame gets wrong pairs but in-range bins, never UB
        img[a] = g.pbc[a] ? __double2int_rd(f) : 0;
        const int ci = __double2int_rz((f - (double)img[a]) * (double)g.ncell[a]);
        c[a] = ci < 0 ? 0 : (ci >= g.ncell[a] ? g.ncell[a] - 1 : ci);
    }
#pragma unroll
    for (int x = 0; x < 3; ++x) w[x] = p[x] - ((double)img[0] * g.h[0][x] + (double)img[1] * g.h[1][x] + (double)img[2] * g.h[2][x]);
}

// bin c (unwrapped, may leave [0, n)) on axis a -> wrapped bin cw and image im; false when the image is not 0 on an open axis
__device__ __forceinline__ bool nl_lattice_axis(const NlLatticeGeom& g, int a, int c, int& cw, int& im) {
    const int n = g.ncell[a];
    im = c >= 0 ? c / n : -((n - 1 - c) / n);
    cw = c - im * n;
    return im == 0 || g.pbc[a];
}

template <typename T, bool FILL>
__device__ __forceinline__ void nl_lattice_walk(const NlLatticeGeom& g, int64_t i, const T* __restrict__ pos, const int32_t* __restrict__ cell_start,
                                                const int32_t* __restrict__ order, int32_t* __restrict__ counts, const int32_t* __restrict__ row_ptr,
                                                int32_t* __restrict__ nbr, T* __restrict__ shift) {
    double wi[3];
    int imgi[3], ci[3];
    nl_lattice_wrap(g, pos, i, wi, imgi, ci);
    int cnt = 0;
    int out = FILL ? row_ptr[i] : 0;  // row_ptr is int32; an int64 cursor spills in the fp32 fill
    for (int dx = -g.reach[0]; dx <= g.reach[0]; ++dx) {
        int cx, ix;
        if (!nl_lattice_axis(g, 0, ci[0] + dx, cx, ix)) continue;
        for (int dy = -g.reach[1]; dy <= g.reach[1]; ++dy) {
            int cy, iy;
            if (!nl_lattice_axis(g, 1, ci[1] + dy, cy, iy)) continue;
            for (int dz = -g.reach[2]; dz <= g.reach[2]; ++dz) {
                int cz, iz;
                if (!nl_lattice_axis(g, 2, ci[2] + dz, cz, iz)) continue;
                // image offset of the visited bin minus the centre: r = wj + off
                double off[3];
#pragma unroll
                for (int x = 0; x < 3; ++x) off[x] = (double)ix * g.h[0][x] + (double)iy * g.h[1][x] + (double)iz * g.h[2][x] - wi[x];
                const bool home = ix == 0 && iy == 0 && iz == 0;
                const int cell = (cx * g.ncell[1] + cy) * g.ncell[2] + cz;
                const int a0 = cell_start[cell], a1 = cell_start[cell + 1];
                for (int a = a0; a < a1; ++a) {
                    const int64_t j = order[a];
                    double wj[3];
                    int imgj[3], cj[3];
                    nl_lattice_wrap(g, pos, j, wj, imgj, cj);
                    double r2 = 0;
#pragma unroll
                    for (int x = 0; x < 3; ++x) {
                        const double rx = wj[x] + off[x];
                        r2 += rx * rx;
                    }
                    if (r2 < g.rmax2 && !(home && j == i)) {
                        if (FILL) {
                            // in double: saturated images must not overflow an int
                            const double s0 = (double)ix - imgj[0] + imgi[0], s1 = (double)iy - imgj[1] + imgi[1], s2 = (double)iz - imgj[2] + imgi[2];
                            nbr[out] = (int32_t)j;
#pragma unroll
                            for (int x = 0; x < 3; ++x) shift[(int64_t)out * 3 + x] = (T)(s0 * g.h[0][x] + s1 * g.h[1][x] + s2 * g.h[2][x]);
                            ++out;
                        }
                        ++cnt;
                    }
                }
            }
        }
    }
    if (!FILL) counts[i] = cnt;
}

template <typename T, bool LATTICE>
__global__ void __launch_bounds__(256) nl_bin_kernel(NlGeomOf<LATTICE> g, int64_t n, const T* __restrict__ pos, int32_t* __restrict__ cell_id) {
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    int img[3], c[3];
    if constexpr (LATTICE) {
        double w[3];
        nl_lattice_wrap(g, pos, i, w, img, c);
    } else {
        T w[3];
        nl_wrap(g, pos, i, w, img, c);
    }
    cell_id[i] = (c[0] * g.ncell[1] + c[1]) * g.ncell[2] + c[2];
}

// FILL = false: counts[i]; FILL = true: nbr / shift rows at row_ptr[i].  LATTICE = false: orthorhombic box, 27 cells
template <typename T, bool FILL, bool LATTICE>
__global__ void __launch_bounds__(128) nl_walk_kernel(NlGeomOf<LATTICE> g, int64_t n_centres, const T* __restrict__ pos,
                                                      const int32_t* __restrict__ cell_start, const int32_t* __restrict__ order,
                                                      int32_t* __restrict__ counts, const int32_t* __restrict__ row_ptr,
                                                      int32_t* __restrict__ nbr, T* __restrict__ shift) {
    const int64_t i = (int64_t)blockIdx.x * 128 + threadIdx.x;
    if (i >= n_centres) return;
    if constexpr (LATTICE) {
        nl_lattice_walk<T, FILL>(g, i, pos, cell_start, order, counts, row_ptr, nbr, shift);
    } else {
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

// Checks and completes a general-lattice grid on the host, in double / int64 before anything is launched.  The
// inverse is computed here so that no caller can pass one inconsistent with the rows.  data.lattice_grid mirrors the
// height and reach arithmetic operation for operation, so the grids it returns pass on the same quotients.
int nl_lattice_geom(NlLatticeGeom& g, const double* rows, const double* origin, const int32_t* pbc, const int32_t* ncell,
                    const int32_t* reach, double r_max) {
    if (!(r_max > 0) || !std::isfinite(r_max)) return 1;
    for (int k = 0; k < 9; ++k) {
        if (!std::isfinite(rows[k])) return 1;
        g.h[k / 3][k % 3] = rows[k];
    }
    double cr[3][3], norm[3];  // cr[a] = h[a+1] x h[a+2]: det . hinv column a
    for (int a = 0; a < 3; ++a) {
        const double* p = g.h[(a + 1) % 3];
        const double* q = g.h[(a + 2) % 3];
        cr[a][0] = p[1] * q[2] - p[2] * q[1];
        cr[a][1] = p[2] * q[0] - p[0] * q[2];
        cr[a][2] = p[0] * q[1] - p[1] * q[0];
        norm[a] = std::sqrt(g.h[a][0] * g.h[a][0] + g.h[a][1] * g.h[a][1] + g.h[a][2] * g.h[a][2]);
    }
    const double det = g.h[0][0] * cr[0][0] + g.h[0][1] * cr[0][1] + g.h[0][2] * cr[0][2];
    // singular (or a cell whose rows are within 1e-12 rad of a common plane)
    if (!std::isfinite(det) || !(std::fabs(det) > 1e-12 * norm[0] * norm[1] * norm[2])) return 2;
    int64_t cells = 1, visits = 1;
    for (int a = 0; a < 3; ++a) {
        if (!std::isfinite(origin[a])) return 1;
        for (int x = 0; x < 3; ++x) g.hinv[x][a] = cr[a][x] / det;
        g.origin[a] = origin[a]; g.pbc[a] = pbc[a] != 0; g.ncell[a] = ncell[a]; g.reach[a] = reach[a];
        if (ncell[a] < 1 || reach[a] < 1) return 3;
        // bin c_a + d of the walk stays an int
        if ((int64_t)ncell[a] + reach[a] >= (int64_t)0x7fffffff) return 4;
        const double height = std::fabs(det) / std::sqrt(cr[a][0] * cr[a][0] + cr[a][1] * cr[a][1] + cr[a][2] * cr[a][2]);
        if (height / ncell[a] * reach[a] < r_max * (1 - 1e-12)) return 5;  // k_a bins of thickness t_a reach r_max
        cells *= ncell[a];
        if (cells >= (int64_t)0x7fffffff) return 6;  // int32 cell ids and cell_start offsets
        visits *= 2 * (int64_t)reach[a] + 1;
        if (visits >= (int64_t)0x7fffffff) return 7;  // bins visited per centre
    }
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
    if (pos_dtype == AB2_F64) nl_bin_kernel<double, false><<<ab2_blocks(n, 256), 256, 0, st>>>(g, n, (const double*)pos, cell_id);
    else nl_bin_kernel<float, false><<<ab2_blocks(n, 256), 256, 0, st>>>(g, n, (const float*)pos, cell_id);
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
        nl_walk_kernel<double, false, false><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const double*)pos, cell_start, order, counts, nullptr, nullptr, nullptr);
    else
        nl_walk_kernel<float, false, false><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const float*)pos, cell_start, order, counts, nullptr, nullptr, nullptr);
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
        nl_walk_kernel<double, true, false><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const double*)pos, cell_start, order, nullptr, row_ptr, nbr, (double*)shift);
    else
        nl_walk_kernel<float, true, false><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const float*)pos, cell_start, order, nullptr, row_ptr, nbr, (float*)shift);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// ---- general lattice ------------------------------------------------------------------------

extern "C" int ab2_nl_lattice_bin(int pos_dtype, int64_t n, const void* pos, const double* rows_host, const double* origin_host,
                                  const int32_t* pbc_host, const int32_t* ncell_host, const int32_t* reach_host, double r_max,
                                  int32_t* cell_id, void* stream) {
    AB2_CHECK_ARG(rows_host && origin_host && pbc_host && ncell_host && reach_host, "null pointer");
    NlLatticeGeom g;
    AB2_CHECK_ARG(nl_lattice_geom(g, rows_host, origin_host, pbc_host, ncell_host, reach_host, r_max) == 0,
                  "cell / bin grid (need finite non-singular rows, >= 1 bin per axis, reach * bin thickness >= r_max, < 2^31 - 1 bins, "
                  "< 2^31 - 1 bins visited per centre)");
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos && cell_id, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    cudaStream_t st = (cudaStream_t)stream;
    if (pos_dtype == AB2_F64) nl_bin_kernel<double, true><<<ab2_blocks(n, 256), 256, 0, st>>>(g, n, (const double*)pos, cell_id);
    else nl_bin_kernel<float, true><<<ab2_blocks(n, 256), 256, 0, st>>>(g, n, (const float*)pos, cell_id);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_nl_lattice_count(int pos_dtype, int64_t n_centres, const void* pos, const double* rows_host, const double* origin_host,
                                    const int32_t* pbc_host, const int32_t* ncell_host, const int32_t* reach_host, double r_max,
                                    const int32_t* cell_start, const int32_t* order, int32_t* counts, void* stream) {
    AB2_CHECK_ARG(rows_host && origin_host && pbc_host && ncell_host && reach_host, "null pointer");
    NlLatticeGeom g;
    AB2_CHECK_ARG(nl_lattice_geom(g, rows_host, origin_host, pbc_host, ncell_host, reach_host, r_max) == 0, "cell / bin grid");
    if (n_centres == 0) return 0;
    AB2_CHECK_ARG(pos && cell_start && order && counts, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    cudaStream_t st = (cudaStream_t)stream;
    if (pos_dtype == AB2_F64)
        nl_walk_kernel<double, false, true><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const double*)pos, cell_start, order, counts, nullptr, nullptr, nullptr);
    else
        nl_walk_kernel<float, false, true><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const float*)pos, cell_start, order, counts, nullptr, nullptr, nullptr);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_nl_lattice_fill(int pos_dtype, int64_t n_centres, const void* pos, const double* rows_host, const double* origin_host,
                                   const int32_t* pbc_host, const int32_t* ncell_host, const int32_t* reach_host, double r_max,
                                   const int32_t* cell_start, const int32_t* order, const int32_t* row_ptr, int32_t* nbr, void* shift,
                                   void* stream) {
    AB2_CHECK_ARG(rows_host && origin_host && pbc_host && ncell_host && reach_host, "null pointer");
    NlLatticeGeom g;
    AB2_CHECK_ARG(nl_lattice_geom(g, rows_host, origin_host, pbc_host, ncell_host, reach_host, r_max) == 0, "cell / bin grid");
    if (n_centres == 0) return 0;
    AB2_CHECK_ARG(pos && cell_start && order && row_ptr && nbr && shift, "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    cudaStream_t st = (cudaStream_t)stream;
    if (pos_dtype == AB2_F64)
        nl_walk_kernel<double, true, true><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const double*)pos, cell_start, order, nullptr, row_ptr, nbr, (double*)shift);
    else
        nl_walk_kernel<float, true, true><<<ab2_blocks(n_centres, 128), 128, 0, st>>>(g, n_centres, (const float*)pos, cell_start, order, nullptr, row_ptr, nbr, (float*)shift);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

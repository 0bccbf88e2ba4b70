// Exchange plan of a 1-D slab decomposition, built on the device from the rank's own atoms (DistributedCalculator's
// rebuild, allegro_b200/halo.py).  Mid-trajectory no rank holds the global frame, so the host cannot make the plan.
//
// One count -> scan -> fill pair in the style of nlist.cu, with two modes:
//   mode 0 (migration): wrap every position into the box on all three axes (image += the whole boxes removed) and
//          classify each atom by its destination slab s = clamp(floor(x / width), 0, world - 1), the rule
//          SlabDecomposition uses: list 0 stays, list 1 goes to the left neighbour, list 2 to the right one; column 3
//          counts atoms bound for a non-adjacent slab, or that moved more than `jump` outside [lo, hi) before the wrap.
//   mode 1 (ghosts): atoms with x < lo + r_list (list 0, sent to the left neighbour) and x >= hi - r_list (list 1, to the
//          right one), compared in fp64.  An atom can be in both lists when the slab is thinner than 2 r_list.
// slab_plan_count writes a class byte per atom and per-block counts [block][4]; the host takes an exclusive prefix sum
// over the blocks (plumbing) and reads the totals once; slab_plan_fill writes the int64 index lists in ascending atom
// order (stable: the order of a list depends on nothing but the atoms' order).
//
// The wrap is x - floor(x / L) L with IEEE division and without fused multiply-add (explicit _rn intrinsics), then one
// correction either way, so that the result is in [0, L) in the positions' own dtype and bitwise what the same three
// operations give in torch (tests/test_halo_gloo_md.py restates them).
//
// The LATTICE instantiation (ab2_slab_plan_count_lattice) cuts any regular cell along lattice row 0, in fractional
// coordinates s = pos . h^-1 (the inverse from lattice.cuh, computed on the host): rank r owns s_0 in [r / world,
// (r + 1) / world).  Mode 0 wraps on all three axes with img_a = floor(s_a) and pos <- pos - sum_a img_a h_a, computed in
// fp64 and rounded once to the positions' dtype, then classifies by clamp(floor(s_0 world), 0, world - 1) of the wrapped
// position; jump is in fractional units and world 2 picks the side by the unwrapped s_0 < lo.  Mode 1 selects
// s_0 < lo + r_list / H_0 and s_0 >= hi - r_list / H_0 (H_0 the height of the cell along row 0).  Every product and sum
// is an explicit _rn operation in a fixed order (s_a = (p_0 hinv_0a + p_1 hinv_1a) + p_2 hinv_2a), so a torch restatement
// (tests/test_halo_gloo_lattice.py) reproduces the kernel bit for bit.
#include <cmath>
#include <type_traits>

#include "common.cuh"
#include "lattice.cuh"

namespace {

constexpr int kPlanBlock = 256;

__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double sub_rn(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }

struct SlabGeom {
    double box[3];
    double width, lo, hi, jump, r_list;
    int rank, world;
};

// fractional geometry of the LATTICE kernels: lo = rank / world, hi = (rank + 1) / world, jump in fractional units,
// low_face = lo + r_list / H_0, high_face = hi - r_list / H_0 (all rounded once on the host)
struct SlabLatticeGeom {
    double h[3][3], hinv[3][3];
    double lo, hi, jump, low_face, high_face;
    int rank, world;
};

template <bool LATTICE>
using SlabGeomOf = std::conditional_t<LATTICE, SlabLatticeGeom, SlabGeom>;

// s_a = (p_0 hinv[0][a] + p_1 hinv[1][a]) + p_2 hinv[2][a], no FMA
__device__ __forceinline__ double frac_rn(const SlabLatticeGeom& g, const double (&p)[3], int a) {
    return add_rn(add_rn(mul_rn(p[0], g.hinv[0][a]), mul_rn(p[1], g.hinv[1][a])), mul_rn(p[2], g.hinv[2][a]));
}

// class bits of one atom: bit k = member of list k (k < 3), bit 3 = refused (mode 0 only)
template <typename T>
__device__ __forceinline__ unsigned slab_class_lattice(const SlabLatticeGeom& g, int mode, T* __restrict__ pos, int32_t* __restrict__ image,
                                                       int64_t i) {
    const double p[3] = {(double)pos[i * 3 + 0], (double)pos[i * 3 + 1], (double)pos[i * 3 + 2]};
    if (mode == 1) {
        const double s0 = frac_rn(g, p, 0);
        return (s0 < g.low_face ? 1u : 0u) | (s0 >= g.high_face ? 2u : 0u);
    }
    double img[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) img[a] = floor(frac_rn(g, p, a));
    const double s0 = frac_rn(g, p, 0);  // unwrapped
    double w[3];
#pragma unroll
    for (int x = 0; x < 3; ++x) {
        const double shift = add_rn(add_rn(mul_rn(img[0], g.h[0][x]), mul_rn(img[1], g.h[1][x])), mul_rn(img[2], g.h[2][x]));
        const T wx = (T)sub_rn(p[x], shift);
        pos[i * 3 + x] = wx;
        w[x] = (double)wx;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) image[i * 3 + a] += (int32_t)img[a];  // saturates for an exploded frame: never UB
    if (s0 < g.lo - g.jump || s0 >= g.hi + g.jump) return 8u;
    int s = __double2int_rd(mul_rn(frac_rn(g, w, 0), (double)g.world));
    s = s < 0 ? 0 : (s >= g.world ? g.world - 1 : s);
    const int d = (s - g.rank + g.world) % g.world;
    if (d == 0) return 1u;
    if (g.world == 2) return s0 < g.lo ? 2u : 4u;  // both neighbours are one rank: the side the atom left by decides
    if (d == g.world - 1) return 2u;
    if (d == 1) return 4u;
    return 8u;
}

template <typename T>
__device__ __forceinline__ unsigned slab_class(const SlabGeom& g, int mode, T* __restrict__ pos, int32_t* __restrict__ image, int64_t i) {
    if (mode == 1) {
        const double x = (double)pos[i * 3];
        return (x < g.lo + g.r_list ? 1u : 0u) | (x >= g.hi - g.r_list ? 2u : 0u);
    }
    const T xr = pos[i * 3];
    T w0 = xr;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const T L = (T)g.box[a];
        const T x = pos[i * 3 + a];
        T img = floor(div_rn(x, L));
        T w = sub_rn(x, mul_rn(img, L));
        if (w < (T)0) { w = add_rn(w, L); img = sub_rn(img, (T)1); }
        if (w >= L) { w = sub_rn(w, L); img = add_rn(img, (T)1); }
        pos[i * 3 + a] = w;
        image[i * 3 + a] += (int32_t)img;  // saturates for an exploded frame: never UB
        if (a == 0) w0 = w;
    }
    const double xd = (double)xr;
    if (xd < g.lo - g.jump || xd >= g.hi + g.jump) return 8u;
    int s = (int)div_rn(w0, (T)g.width);
    s = s < 0 ? 0 : (s >= g.world ? g.world - 1 : s);
    const int d = (s - g.rank + g.world) % g.world;
    if (d == 0) return 1u;
    if (g.world == 2) return xd < g.lo ? 2u : 4u;  // both neighbours are one rank: the side the atom left by decides
    if (d == g.world - 1) return 2u;
    if (d == 1) return 4u;
    return 8u;
}

template <typename T, bool LATTICE>
__global__ void __launch_bounds__(kPlanBlock) slab_plan_count_kernel(SlabGeomOf<LATTICE> g, int mode, int64_t n, T* __restrict__ pos,
                                                                     int32_t* __restrict__ image, uint8_t* __restrict__ cls,
                                                                     int32_t* __restrict__ block_counts) {
    __shared__ int cnt[4];
    if (threadIdx.x < 4) cnt[threadIdx.x] = 0;
    __syncthreads();
    const int64_t i = (int64_t)blockIdx.x * kPlanBlock + threadIdx.x;
    unsigned c = 0;
    if (i < n) {
        if constexpr (LATTICE) c = slab_class_lattice(g, mode, pos, image, i);
        else c = slab_class(g, mode, pos, image, i);
        cls[i] = (uint8_t)c;
    }
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const unsigned m = __ballot_sync(0xffffffffu, (c >> k) & 1u);
        if (lane == 0 && m) atomicAdd(&cnt[k], __popc(m));
    }
    __syncthreads();
    if (threadIdx.x < 4) block_counts[(int64_t)blockIdx.x * 4 + threadIdx.x] = cnt[threadIdx.x];
}

// lists[k][offsets[block][k] + rank of atom i among the block's members of list k] = i, for the lists that are not null
__global__ void __launch_bounds__(kPlanBlock) slab_plan_fill_kernel(int64_t n, const uint8_t* __restrict__ cls, const int32_t* __restrict__ offsets,
                                                                    int64_t* __restrict__ l0, int64_t* __restrict__ l1, int64_t* __restrict__ l2) {
    constexpr int kWarps = kPlanBlock / 32;
    __shared__ int warp_cnt[3][kWarps];
    const int64_t i = (int64_t)blockIdx.x * kPlanBlock + threadIdx.x;
    const unsigned c = i < n ? cls[i] : 0u;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned below = (1u << lane) - 1u;
    unsigned mask[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        mask[k] = __ballot_sync(0xffffffffu, (c >> k) & 1u);
        if (lane == 0) warp_cnt[k][warp] = __popc(mask[k]);
    }
    __syncthreads();
    int64_t* lists[3] = {l0, l1, l2};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (!((c >> k) & 1u) || lists[k] == nullptr) continue;
        int pos = offsets[(int64_t)blockIdx.x * 4 + k] + __popc(mask[k] & below);
        for (int w = 0; w < warp; ++w) pos += warp_cnt[k][w];
        lists[k][pos] = i;
    }
}

int slab_geom(SlabGeom& g, const double* box, int rank, int world, double width, double jump, double r_list) {
    for (int a = 0; a < 3; ++a) {
        if (!(box[a] > 0) || !std::isfinite(box[a])) return 1;
        g.box[a] = box[a];
    }
    if (world < 1 || rank < 0 || rank >= world || !(width > 0) || !(jump >= 0) || !(r_list >= 0)) return 2;
    g.rank = rank; g.world = world; g.width = width; g.jump = jump; g.r_list = r_list;
    g.lo = rank * width;
    g.hi = (rank + 1) * width;
    return 0;
}

}  // namespace

extern "C" int ab2_slab_plan_count(int pos_dtype, int mode, int64_t n, void* pos, int32_t* image, const double* box_host, int rank, int world,
                                   double width, double jump, double r_list, uint8_t* cls, int32_t* block_counts, void* stream) {
    AB2_CHECK_ARG(box_host && (mode == 0 || mode == 1) && n >= 0, "bad arguments");
    SlabGeom g;
    AB2_CHECK_ARG(slab_geom(g, box_host, rank, world, width, jump, r_list) == 0,
                  "slab geometry (need finite box lengths > 0, 0 <= rank < world, width > 0, jump >= 0, r_list >= 0)");
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos && cls && block_counts && (mode == 1 || image), "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = ab2_blocks(n, kPlanBlock);
    if (pos_dtype == AB2_F64)
        slab_plan_count_kernel<double, false><<<grid, kPlanBlock, 0, st>>>(g, mode, n, (double*)pos, image, cls, block_counts);
    else
        slab_plan_count_kernel<float, false><<<grid, kPlanBlock, 0, st>>>(g, mode, n, (float*)pos, image, cls, block_counts);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_slab_plan_count_lattice(int pos_dtype, int mode, int64_t n, void* pos, int32_t* image, const double* rows_host, int rank,
                                           int world, double jump, double r_list, uint8_t* cls, int32_t* block_counts, void* stream) {
    AB2_CHECK_ARG(rows_host && (mode == 0 || mode == 1) && n >= 0, "bad arguments");
    Ab2Lattice lat;
    AB2_CHECK_ARG(ab2_lattice_inverse(rows_host, lat) == 0, "cell (need finite rows, not singular or within 1e-12 rad of a common plane)");
    AB2_CHECK_ARG(world >= 1 && rank >= 0 && rank < world && jump >= 0 && r_list >= 0 && std::isfinite(r_list),
                  "slab geometry (need 0 <= rank < world, jump >= 0, finite r_list >= 0)");
    SlabLatticeGeom g;
    for (int a = 0; a < 3; ++a)
        for (int x = 0; x < 3; ++x) {
            g.h[a][x] = lat.h[a][x];
            g.hinv[a][x] = lat.hinv[a][x];
        }
    g.rank = rank; g.world = world; g.jump = jump;
    g.lo = (double)rank / world;
    g.hi = (double)(rank + 1) / world;
    const double r_frac = r_list / ab2_lattice_height(lat, 0);
    g.low_face = g.lo + r_frac;
    g.high_face = g.hi - r_frac;
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos && cls && block_counts && (mode == 1 || image), "null pointer");
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = ab2_blocks(n, kPlanBlock);
    if (pos_dtype == AB2_F64)
        slab_plan_count_kernel<double, true><<<grid, kPlanBlock, 0, st>>>(g, mode, n, (double*)pos, image, cls, block_counts);
    else
        slab_plan_count_kernel<float, true><<<grid, kPlanBlock, 0, st>>>(g, mode, n, (float*)pos, image, cls, block_counts);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_slab_plan_fill(int64_t n, const uint8_t* cls, const int32_t* block_offsets, int64_t* list0, int64_t* list1, int64_t* list2,
                                  void* stream) {
    AB2_CHECK_ARG(n >= 0, "bad arguments");
    if (n == 0) return 0;
    AB2_CHECK_ARG(cls && block_offsets, "null pointer");
    slab_plan_fill_kernel<<<ab2_blocks(n, kPlanBlock), kPlanBlock, 0, (cudaStream_t)stream>>>(n, cls, block_offsets, list0, list1, list2);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

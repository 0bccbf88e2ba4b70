// The per-frame all-pairs walk of nlist_frames.cu, shared with the fixed-slot rebuild of nlist_slots.cu.
//
// One warp per centre.  The lanes take 32 consecutive atoms of the centre's own frame at a time (coalesced reads) and
// every lane walks its atom over the frame's image range; the fill pass places the lanes' hits with a warp prefix sum.
// So a row is ordered by neighbour index, then by image (x, y, z) lexicographically: the order of
// data.neighbor_list(..., method="brute").
//
// Geometry per frame, all on the device: cell[b] (rows = lattice vectors), its inverse, pbc[b][3] and nimg[b][3].  Positions
// are wrapped into the cell along the periodic axes in fractional coordinates (frac = pos @ inv, image = floor(frac)), and
// the raw image offsets are folded back into the shift, so  r = pos[nbr] + shift - pos[ctr]  holds for the RAW positions.
// An axis a needs n_a = ceil(r_max / h_a) images on each side, h_a = |det cell| / |b x c| the cell height along that axis;
// the host computes n_a (_lib.nl_frames through data.frames_geometry, in fp64 from the cell as rounded to the positions'
// dtype), refuses near-singular cells and bounds the images per pair, so the walk below is bounded by what it is given.
// A frame with no periodic axis is searched as it is (no wrap, one image): a molecule.
#pragma once
#include "common.cuh"

namespace {

constexpr int NLF_WARPS = 4;  // warps (centres) per CTA

// largest b in [0, B) with frame_ptr[b] <= i  (the frame of atom i; empty frames are skipped)
__device__ __forceinline__ int64_t nlf_frame_of(const int32_t* __restrict__ frame_ptr, int64_t B, int64_t i) {
    int64_t lo = 0, hi = B - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (frame_ptr[mid] <= i) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

template <typename T>
struct NlfFrame {
    T c[9], inv[9];
    int pbc[3], nimg[3];
    bool periodic;
};

template <typename T>
__device__ __forceinline__ void nlf_load_frame(NlfFrame<T>& f, const T* __restrict__ cell, const T* __restrict__ inv,
                                               const int32_t* __restrict__ pbc, const int32_t* __restrict__ nimg, int64_t b) {
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        f.c[k] = cell[b * 9 + k];
        f.inv[k] = inv[b * 9 + k];
    }
    f.periodic = false;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        f.pbc[a] = pbc[b * 3 + a] != 0;
        f.periodic |= f.pbc[a];
        f.nimg[a] = f.pbc[a] ? nimg[b * 3 + a] : 0;  // images on each side (host: ceil(r_max / height))
    }
}

// wrapped position and raw image of atom j (the host of data._brute_force: frac = pos @ inv, img = floor on periodic axes)
template <typename T>
__device__ __forceinline__ void nlf_wrap(const NlfFrame<T>& f, const T* __restrict__ pos, int64_t j, T (&w)[3], int (&img)[3]) {
    const T p[3] = {pos[j * 3 + 0], pos[j * 3 + 1], pos[j * 3 + 2]};
    if (!f.periodic) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            w[a] = p[a];
            img[a] = 0;
        }
        return;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const T fr = p[0] * f.inv[0 * 3 + k] + p[1] * f.inv[1 * 3 + k] + p[2] * f.inv[2 * 3 + k];
        img[k] = f.pbc[k] ? (int)floor(fr) : 0;
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
        w[a] = p[a] - ((T)img[0] * f.c[0 * 3 + a] + (T)img[1] * f.c[1 * 3 + a] + (T)img[2] * f.c[2 * 3 + a]);
}

// calls hit(sx, sy, sz) for every image s (lexicographic order) under which atom j is a neighbour of centre i
template <typename T, typename F>
__device__ __forceinline__ void nlf_images(const NlfFrame<T>& f, const T (&wi)[3], const T (&wj)[3], bool self, T r_max, F&& hit) {
    for (int sx = -f.nimg[0]; sx <= f.nimg[0]; ++sx)
        for (int sy = -f.nimg[1]; sy <= f.nimg[1]; ++sy)
            for (int sz = -f.nimg[2]; sz <= f.nimg[2]; ++sz) {
                if (self && sx == 0 && sy == 0 && sz == 0) continue;
                T r2 = 0;
#pragma unroll
                for (int a = 0; a < 3; ++a) {
                    const T off = (T)sx * f.c[0 * 3 + a] + (T)sy * f.c[1 * 3 + a] + (T)sz * f.c[2 * 3 + a];
                    const T d = (wj[a] + off) - wi[a];
                    r2 += d * d;
                }
                if (sqrt(r2) < r_max) hit(sx, sy, sz);
            }
}

// FILL = false: counts[i] = neighbours of centre i;  FILL = true: nbr / shift of those neighbours at row_ptr[i] on.
// SLOTS (nlist_slots.cu): only the frames with frame_flag[b] == 1 are walked (the others leave at once), and the fill
// also writes ctr over the whole row [row_ptr[i], row_ptr[i+1]), pads the row after its real edges with self-edges
// shifted by (pad, 0, 0), and copies pos[i] to pos_ref[i].  The SLOTS arguments are unused (and may be null) otherwise.
template <typename T, bool FILL, bool SLOTS = false>
__global__ void __launch_bounds__(NLF_WARPS * 32) nlf_walk_kernel(int64_t n, int64_t B, const int32_t* __restrict__ frame_ptr,
                                                                  const T* __restrict__ pos, const T* __restrict__ cell,
                                                                  const T* __restrict__ inv, const int32_t* __restrict__ pbc,
                                                                  const int32_t* __restrict__ nimg, double r_max, int32_t* __restrict__ counts,
                                                                  const int32_t* __restrict__ row_ptr, int32_t* __restrict__ nbr,
                                                                  T* __restrict__ shift, const int32_t* __restrict__ frame_flag = nullptr,
                                                                  int32_t* __restrict__ ctr = nullptr, T* __restrict__ pos_ref = nullptr,
                                                                  double pad = 0.0) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * NLF_WARPS + (threadIdx.x >> 5);
    if (i >= n) return;  // whole warps leave together
    const int64_t b = nlf_frame_of(frame_ptr, B, i);
    if constexpr (SLOTS) {
        if (frame_flag[b] != 1) return;  // frame not flagged for a rebuild, or its slot overflowed: nothing to write
    }
    const int64_t j0 = frame_ptr[b], j1 = frame_ptr[b + 1];
    NlfFrame<T> f;
    nlf_load_frame(f, cell, inv, pbc, nimg, b);
    T wi[3];
    int imgi[3];
    nlf_wrap(f, pos, i, wi, imgi);
    const T rc = (T)r_max;
    int64_t out = FILL ? (int64_t)row_ptr[i] : 0;
    int total = 0;
    for (int64_t base = j0; base < j1; base += 32) {
        const int64_t j = base + lane;
        T wj[3];
        int imgj[3];
        int cnt = 0;
        if (j < j1) {
            nlf_wrap(f, pos, j, wj, imgj);
            nlf_images(f, wi, wj, j == i, rc, [&](int, int, int) { ++cnt; });
        }
        if (!FILL) {
            total += cnt;
            continue;
        }
        // exclusive prefix of the lanes' hit counts: lane order = neighbour order
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        const int chunk = __shfl_sync(0xffffffffu, incl, 31);
        if (cnt) {
            int64_t k = out + incl - cnt;
            nlf_images(f, wi, wj, j == i, rc, [&](int sx, int sy, int sz) {
                const int r0 = sx - imgj[0] + imgi[0], r1 = sy - imgj[1] + imgi[1], r2 = sz - imgj[2] + imgi[2];
                nbr[k] = (int32_t)j;
#pragma unroll
                for (int a = 0; a < 3; ++a)
                    shift[k * 3 + a] = (T)r0 * f.c[0 * 3 + a] + (T)r1 * f.c[1 * 3 + a] + (T)r2 * f.c[2 * 3 + a];
                ++k;
            });
        }
        out += chunk;
    }
    if (!FILL) {
        total = warp_sum(total);
        if (lane == 0) counts[i] = total;
    }
    if constexpr (SLOTS && FILL) {
        // out = the end of the row's real edges; the rest of the row is padding
        const int64_t r1 = row_ptr[i + 1];
        for (int64_t k = (int64_t)row_ptr[i] + lane; k < r1; k += 32) {
            ctr[k] = (int32_t)i;
            if (k >= out) {
                nbr[k] = (int32_t)i;
                shift[k * 3 + 0] = (T)pad;
                shift[k * 3 + 1] = (T)0;
                shift[k * 3 + 2] = (T)0;
            }
        }
        if (lane < 3) pos_ref[i * 3 + lane] = pos[i * 3 + lane];
    }
}

}  // namespace

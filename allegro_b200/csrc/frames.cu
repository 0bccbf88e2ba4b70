// Per-frame reductions of a batch of frames concatenated into one graph: the total energy of every frame, its virial and
// its potential heat current (sums), and the max / min / mean of a per-atom value (the committee's force deviation).
//
// A batch may hold one frame of several million edges next to thousands of frames of ten edges, and the result of a frame
// may depend neither on the launch nor on the other frames.  So every frame is cut into fixed chunks of FR_CHUNK
// elements counted from ITS OWN start; one CTA reduces one chunk in a fixed order (thread t takes elements t, t + 256, ...
// of the chunk, then a fixed warp / block tree), and a second kernel adds a frame's chunk partials in chunk order.
// No float atomics; an empty frame gives an exact zero.
//
// Chunk ids without a prefix sum over the frames: frame b owns the ids [v_b, v_{b+1}) with v_b = start_b / FR_CHUNK + b.
// Since start_{b+1} = start_b + len_b,  v_{b+1} - v_b >= ceil(len_b / FR_CHUNK): every frame's chunks fit in its range,
// and all ids lie below total / FR_CHUNK + B (the grid of the first kernel, and the scratch size).  The CTA of id v finds
// its frame by a binary search over the (strictly increasing) v_b; ids past a frame's last chunk do nothing.
#include "common.cuh"

namespace {

constexpr int FR_CHUNK = 2048;
constexpr int FR_THREADS = 256;

// start of frame b's element range: frame_ptr[b] for per-atom data, row_ptr[frame_ptr[b]] for per-edge data
__device__ __forceinline__ int64_t fr_start(const int32_t* __restrict__ frame_ptr, const int32_t* __restrict__ row_ptr, int64_t b) {
    const int32_t a = frame_ptr[b];
    return row_ptr ? (int64_t)row_ptr[a] : (int64_t)a;
}

__device__ __forceinline__ int64_t fr_vid(const int32_t* frame_ptr, const int32_t* row_ptr, int64_t b) {
    return fr_start(frame_ptr, row_ptr, b) / FR_CHUNK + b;
}

// The reduction operator.  FR_SUM: every one of the W values is a sum.  FR_EXTREMA (W = 3): value 0 is the max, value 1
// the min and value 2 the sum of x[e]; the combine turns the sum into the mean over the frame's elements.
enum { FR_SUM = 0, FR_EXTREMA = 1 };

// identity of value k: 0 for a sum, -inf / +inf for the max / min
template <int OP>
__device__ __forceinline__ double fr_ident(int k) {
    if constexpr (OP == FR_EXTREMA) {
        if (k == 0) return -INFINITY;
        if (k == 1) return INFINITY;
    }
    return 0.0;
}

template <int OP>
__device__ __forceinline__ double fr_join(int k, double a, double b) {
    if constexpr (OP == FR_EXTREMA) {
        if (k == 0) return fmax(a, b);
        if (k == 1) return fmin(a, b);
    }
    return a + b;
}

template <int OP>
__device__ __forceinline__ double fr_warp(int k, double v) {
    if constexpr (OP == FR_SUM) {
        return warp_sum(v);
    } else {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = fr_join<OP>(k, v, __shfl_xor_sync(0xffffffffu, v, o));
        return v;
    }
}

// W values per element: W = 1, out += x[e];  W = 9, out[a][c] += vec[e][a] * gvec[e][c] (x = vec, y = gvec);
// W = 3, out[a] += e[e] v[e][a] + sum_c m[e][a][c] v[e][c]  (x = e_atom, y = vel, m = per-atom virial);
// OP = FR_EXTREMA (W = 3): max, min and sum of x[e]
template <typename T, int W, int OP = FR_SUM>
__global__ void __launch_bounds__(FR_THREADS) fr_partial_kernel(int64_t B, const int32_t* __restrict__ frame_ptr,
                                                                const int32_t* __restrict__ row_ptr, const T* __restrict__ x,
                                                                const T* __restrict__ y, const T* __restrict__ m,
                                                                double* __restrict__ part) {
    const int64_t v = blockIdx.x;
    int64_t lo = 0, hi = B - 1;
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (fr_vid(frame_ptr, row_ptr, mid) <= v) lo = mid;
        else hi = mid - 1;
    }
    const int64_t b = lo;
    const int64_t s0 = fr_start(frame_ptr, row_ptr, b), s1 = fr_start(frame_ptr, row_ptr, b + 1);
    const int64_t e0 = s0 + (v - fr_vid(frame_ptr, row_ptr, b)) * FR_CHUNK;
    if (e0 >= s1) return;  // past the frame's last chunk (or an empty frame): no partial, the combine does not read it
    const int64_t e1 = min(e0 + (int64_t)FR_CHUNK, s1);
    double acc[W];
#pragma unroll
    for (int k = 0; k < W; ++k) acc[k] = fr_ident<OP>(k);
    for (int64_t e = e0 + threadIdx.x; e < e1; e += FR_THREADS) {
        if constexpr (OP == FR_EXTREMA) {
            const double a = (double)x[e];
            acc[0] = fmax(acc[0], a);
            acc[1] = fmin(acc[1], a);
            acc[2] += a;
        } else if (W == 1) {
            acc[0] += (double)x[e];
        } else if (W == 3) {
            const double ea = (double)x[e];
            const double v[3] = {(double)y[e * 3 + 0], (double)y[e * 3 + 1], (double)y[e * 3 + 2]};
#pragma unroll
            for (int p = 0; p < 3; ++p) {
                double s = ea * v[p];
#pragma unroll
                for (int q = 0; q < 3; ++q) s += (double)m[e * 9 + p * 3 + q] * v[q];
                acc[p] += s;
            }
        } else {
            const double a[3] = {(double)x[e * 3 + 0], (double)x[e * 3 + 1], (double)x[e * 3 + 2]};
            const double g[3] = {(double)y[e * 3 + 0], (double)y[e * 3 + 1], (double)y[e * 3 + 2]};
#pragma unroll
            for (int p = 0; p < 3; ++p)
#pragma unroll
                for (int q = 0; q < 3; ++q) acc[p * 3 + q] += a[p] * g[q];
        }
    }
    __shared__ double red[FR_THREADS / 32][W];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < W; ++k) {
        const double s = fr_warp<OP>(k, acc[k]);
        if (lane == 0) red[warp][k] = s;
    }
    __syncthreads();
    if (threadIdx.x < W) {
        double s = fr_ident<OP>(threadIdx.x);
#pragma unroll
        for (int w = 0; w < FR_THREADS / 32; ++w) s = fr_join<OP>(threadIdx.x, s, red[w][threadIdx.x]);
        part[v * W + threadIdx.x] = s;
    }
}

// out[b * W + k] = sum over frame b's chunks, in chunk order, of the partials (0 for an empty frame); FR_EXTREMA: max,
// min, and the sum over the frame's length (0, 0, 0 for an empty frame)
template <typename T, int W, int OP = FR_SUM>
__global__ void __launch_bounds__(256) fr_combine_kernel(int64_t B, const int32_t* __restrict__ frame_ptr,
                                                         const int32_t* __restrict__ row_ptr, const double* __restrict__ part,
                                                         T* __restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= B * W) return;
    const int64_t b = t / W;
    const int k = (int)(t - b * W);
    const int64_t len = fr_start(frame_ptr, row_ptr, b + 1) - fr_start(frame_ptr, row_ptr, b);
    const int64_t v0 = fr_vid(frame_ptr, row_ptr, b);
    const int64_t nch = (len + FR_CHUNK - 1) / FR_CHUNK;
    double s = fr_ident<OP>(k);
    for (int64_t c = 0; c < nch; ++c) s = fr_join<OP>(k, s, part[(v0 + c) * W + k]);
    if constexpr (OP == FR_EXTREMA) {
        if (len == 0) s = 0.0;
        else if (k == 2) s = s / (double)len;
    }
    out[t] = (T)s;
}

template <int W, int OP = FR_SUM>
int fr_run(int acc_dtype, int64_t total, int64_t B, const int32_t* frame_ptr, const int32_t* row_ptr, const void* x, const void* y,
           const void* m, double* scratch, int64_t scratch_elems, void* out, void* stream) {
    if (B == 0) return 0;
    AB2_CHECK_ARG(acc_dtype == AB2_F64 || acc_dtype == AB2_F32, "values must be fp64 or fp32");
    constexpr bool sum = OP == FR_SUM;
    AB2_CHECK_ARG(frame_ptr && out && (total == 0 || (x && scratch)) && (W == 1 || !sum || total == 0 || y) &&
                      (W != 3 || !sum || total == 0 || m),
                  "null pointer");
    AB2_CHECK_ARG(total >= 0 && B > 0, "sizes");
    const int64_t nv = total / FR_CHUNK + B;
    AB2_CHECK_ARG(total == 0 || scratch_elems >= nv * W, "scratch smaller than ab2_frame_scratch_elems(total, n_frames) * width");
    AB2_CHECK_ARG(nv <= 0x7fffffffLL, "too many chunks for one launch");
    cudaStream_t st = (cudaStream_t)stream;
    if (acc_dtype == AB2_F64) {
        if (total > 0)
            fr_partial_kernel<double, W, OP><<<(unsigned)nv, FR_THREADS, 0, st>>>(B, frame_ptr, row_ptr, (const double*)x, (const double*)y,
                                                                             (const double*)m, scratch);
        fr_combine_kernel<double, W, OP><<<ab2_blocks(B * W, 256), 256, 0, st>>>(B, frame_ptr, row_ptr, scratch, (double*)out);
    } else {
        if (total > 0)
            fr_partial_kernel<float, W, OP><<<(unsigned)nv, FR_THREADS, 0, st>>>(B, frame_ptr, row_ptr, (const float*)x, (const float*)y,
                                                                            (const float*)m, scratch);
        fr_combine_kernel<float, W, OP><<<ab2_blocks(B * W, 256), 256, 0, st>>>(B, frame_ptr, row_ptr, scratch, (float*)out);
    }
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

}  // namespace

extern "C" int64_t ab2_frame_scratch_elems(int64_t total, int64_t n_frames) { return total / FR_CHUNK + n_frames; }

extern "C" int ab2_frame_sum(int acc_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* x, double* scratch,
                             int64_t scratch_elems, void* out, void* stream) {
    return fr_run<1>(acc_dtype, n, n_frames, frame_ptr, nullptr, x, nullptr, nullptr, scratch, scratch_elems, out, stream);
}

extern "C" int ab2_frame_virial(int acc_dtype, int64_t E, int64_t n_frames, const int32_t* frame_ptr, const int32_t* row_ptr,
                                const void* vec, const void* gvec, double* scratch, int64_t scratch_elems, void* W, void* stream) {
    AB2_CHECK_ARG(row_ptr != nullptr, "null row_ptr");
    return fr_run<9>(acc_dtype, E, n_frames, frame_ptr, row_ptr, vec, gvec, nullptr, scratch, scratch_elems, W, stream);
}

extern "C" int ab2_frame_heat_current(int acc_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* e_atom,
                                      const void* vel, const void* W, double* scratch, int64_t scratch_elems, void* J, void* stream) {
    return fr_run<3>(acc_dtype, n, n_frames, frame_ptr, nullptr, e_atom, vel, W, scratch, scratch_elems, J, stream);
}

extern "C" int ab2_frame_extrema(int acc_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* x, double* scratch,
                                 int64_t scratch_elems, void* out, void* stream) {
    return fr_run<3, FR_EXTREMA>(acc_dtype, n, n_frames, frame_ptr, nullptr, x, nullptr, nullptr, scratch, scratch_elems, out, stream);
}

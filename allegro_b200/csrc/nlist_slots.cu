// Verlet lists of a batch of small frames kept in fixed edge slots, rebuilt frame by frame on the device inside a
// replayed CUDA graph (calculator.BatchedCalculator).
//
// Frame b owns the edges [slot_ptr[b], slot_ptr[b+1]) of one list whose length never changes, so a graph captured on
// the list stays valid while single frames rebuild.  Its atoms' rows partition the slot: each row holds its real edges
// (the rows of nlist_frames.cu, in the same order) and then padding self-edges shifted by (pad, 0, 0), |pad| >= 2 r_list,
// which contribute exactly zero to the model.  The slack of a frame is spread over its atoms: with k = capacity - count
// and n_b atoms, atom l gets k / n_b + (l < k % n_b) padding edges.
//
// One rebuild, every launch with a grid fixed by n and n_frames (graph-capturable; frames not flagged leave at once):
//   slots_check     : frame_flag[b] = 1 when an atom of b moved more than skin / 2 since its frame's last build
//   slots_count     : the nlist_frames.cu count walk, for flagged frames
//   slots_place     : one CTA per flagged frame: capacity check, then row_ptr over the slot (or overflow, nothing written)
//   slots_fill      : the nlist_frames.cu fill walk + ctr, padding and pos_ref, for flagged frames
//   slots_transpose : one CTA per flagged frame: stable counting sort of the slot by neighbour -> col_ptr / col_perm;
//                     clears frame_flag for the next rebuild
#include "nlist_frames.cuh"

namespace {

constexpr int SLOT_PLACE_THREADS = 1024;                             // one CTA per frame: 4 atoms per thread
constexpr int SLOT_ATOMS_PER_THREAD = AB2_FRAMES_MAX_ATOMS / SLOT_PLACE_THREADS;
constexpr int SLOT_T_WARPS = 8;                                      // transpose: warps per frame, each its own histogram
constexpr int SLOT_CHECK_THREADS = 256;

static_assert(SLOT_ATOMS_PER_THREAD * SLOT_PLACE_THREADS == AB2_FRAMES_MAX_ATOMS, "place covers a frame in one pass");

// d2 = (dx * dx + dy * dy) + dz * dz without contraction, so a restatement gets the same bits
__device__ __forceinline__ float slot_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double slot_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float slot_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double slot_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float slot_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double slot_sub(double a, double b) { return __dsub_rn(a, b); }

template <typename T>
__global__ void __launch_bounds__(SLOT_CHECK_THREADS) slots_check_kernel(int64_t n, int64_t B, const int32_t* __restrict__ frame_ptr,
                                                                         const T* __restrict__ pos, const T* __restrict__ pos_ref,
                                                                         T half_skin, int32_t* __restrict__ frame_flag) {
    const int64_t i = (int64_t)blockIdx.x * SLOT_CHECK_THREADS + threadIdx.x;
    if (i >= n) return;
    const T dx = slot_sub(pos[i * 3 + 0], pos_ref[i * 3 + 0]);
    const T dy = slot_sub(pos[i * 3 + 1], pos_ref[i * 3 + 1]);
    const T dz = slot_sub(pos[i * 3 + 2], pos_ref[i * 3 + 2]);
    const T d2 = slot_add(slot_add(slot_mul(dx, dx), slot_mul(dy, dy)), slot_mul(dz, dz));
    if (sqrt(d2) > half_skin) frame_flag[nlf_frame_of(frame_ptr, B, i)] = 1;  // idempotent: any order gives the same flags
}

// exclusive prefix over the CTA of one value per thread (blockDim.x a multiple of 32, at most 1024); returns the
// thread's exclusive prefix and writes the CTA total to *total.  `warp_tot` holds 32 entries.
template <typename V>
__device__ __forceinline__ V slot_block_scan(V v, V* warp_tot, V* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    V incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const V u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        V w = lane < nw ? warp_tot[lane] : V(0);
        V wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const V u = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += u;
        }
        if (lane < nw) warp_tot[lane] = wi - w;
        if (lane == 31) *total = wi;
    }
    __syncthreads();
    const V r = warp_tot[warp] + incl - v;
    __syncthreads();  // warp_tot may be reused by the caller
    return r;
}

__global__ void __launch_bounds__(SLOT_PLACE_THREADS) slots_place_kernel(const int32_t* __restrict__ frame_ptr, const int32_t* __restrict__ slot_ptr,
                                                                         const int32_t* __restrict__ counts, int32_t* __restrict__ frame_flag,
                                                                         int32_t* __restrict__ row_ptr, int32_t* __restrict__ overflow,
                                                                         int32_t* __restrict__ rebuilds) {
    __shared__ long long s_warp[32];
    __shared__ long long s_total;
    const int64_t b = blockIdx.x;
    if (frame_flag[b] != 1) return;  // the whole CTA leaves
    const int64_t a0 = frame_ptr[b], nb = frame_ptr[b + 1] - a0;
    const int64_t s0 = slot_ptr[b], cap = slot_ptr[b + 1] - s0;
    const int t = threadIdx.x;
    // atoms [t * 4, t * 4 + 4) of the frame: consecutive, so the scan below is in atom order
    int c[SLOT_ATOMS_PER_THREAD];
    long long mine = 0;
#pragma unroll
    for (int q = 0; q < SLOT_ATOMS_PER_THREAD; ++q) {
        const int64_t l = (int64_t)t * SLOT_ATOMS_PER_THREAD + q;
        c[q] = l < nb ? counts[a0 + l] : 0;
        mine += c[q];
    }
    slot_block_scan<long long>(mine, s_warp, &s_total);
    const long long count = s_total;
    if (count > cap) {  // uniform over the CTA: the frame keeps its old rows and the host re-sizes every slot
        if (t == 0) {
            atomicAdd(overflow, 1);
            frame_flag[b] = 2;
        }
        return;
    }
    if (nb > 0) {
        const long long k = cap - count, per = k / nb, rest = k % nb;
        long long len[SLOT_ATOMS_PER_THREAD];
        long long sum = 0;
#pragma unroll
        for (int q = 0; q < SLOT_ATOMS_PER_THREAD; ++q) {
            const int64_t l = (int64_t)t * SLOT_ATOMS_PER_THREAD + q;
            len[q] = l < nb ? c[q] + per + (l < rest ? 1 : 0) : 0;
            sum += len[q];
        }
        long long off = slot_block_scan<long long>(sum, s_warp, &s_total);
#pragma unroll
        for (int q = 0; q < SLOT_ATOMS_PER_THREAD; ++q) {
            const int64_t l = (int64_t)t * SLOT_ATOMS_PER_THREAD + q;
            if (l < nb) row_ptr[a0 + l] = (int32_t)(s0 + off);  // row_ptr[frame_ptr[b+1]] = slot_ptr[b+1] is never written
            off += len[q];
        }
    }
    if (t == 0) rebuilds[b] += 1;
}

// Stable counting sort of frame b's slot by neighbour.  Warp w takes the w-th contiguous segment of the slot and keeps
// its own histogram hist[w][0..nb): the columns' per-warp counts are scanned over (column, warp), so warp w's edges of
// column j start after those of warps < w, and inside a warp's segment a chunk of 32 edges is ranked with __match_any_sync
// in lane (= edge) order.  So every column lists its edges in ascending edge id: the order of EdgeCSR.transposed.
__global__ void __launch_bounds__(SLOT_T_WARPS * 32) slots_transpose_kernel(const int32_t* __restrict__ frame_ptr, const int32_t* __restrict__ slot_ptr,
                                                                            const int32_t* __restrict__ nbr, int32_t* __restrict__ frame_flag,
                                                                            int32_t* __restrict__ col_ptr, int32_t* __restrict__ col_perm) {
    extern __shared__ int32_t s_hist[];  // [SLOT_T_WARPS][nb], then the column totals [nb]
    __shared__ int32_t s_warp[32];
    __shared__ int32_t s_total;
    const int64_t b = blockIdx.x;
    const int flag = frame_flag[b];
    if (flag == 0) return;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    if (flag == 1) {
        const int a0 = frame_ptr[b], nb = frame_ptr[b + 1] - a0;
        const int s0 = slot_ptr[b], s1 = slot_ptr[b + 1];
        int32_t* tot = s_hist + SLOT_T_WARPS * nb;
        for (int k = t; k < SLOT_T_WARPS * nb; k += blockDim.x) s_hist[k] = 0;
        __syncthreads();
        const int seg = (s1 - s0 + SLOT_T_WARPS - 1) / SLOT_T_WARPS;
        const int lo = min(s0 + w * seg, s1), hi = min(lo + seg, s1);
        int32_t* h = s_hist + w * nb;
        for (int z = lo + lane; z < hi; z += 32) atomicAdd(&h[nbr[z] - a0], 1);
        __syncthreads();
        for (int j = t; j < nb; j += blockDim.x) {
            int run = 0;
#pragma unroll
            for (int v = 0; v < SLOT_T_WARPS; ++v) {
                const int x = s_hist[v * nb + j];
                s_hist[v * nb + j] = run;
                run += x;
            }
            tot[j] = run;
        }
        __syncthreads();
        // exclusive scan of the column totals, in chunks of blockDim.x columns
        int carry = 0;
        for (int base = 0; base < nb; base += blockDim.x) {
            const int j = base + t;
            const int v = j < nb ? tot[j] : 0;
            const int ex = slot_block_scan<int>(v, s_warp, &s_total) + carry;
            if (j < nb) {
                col_ptr[a0 + j] = s0 + ex;  // col_ptr[frame_ptr[b+1]] = slot_ptr[b+1] is never written
#pragma unroll
                for (int u = 0; u < SLOT_T_WARPS; ++u) s_hist[u * nb + j] += s0 + ex;
            }
            carry += s_total;
            __syncthreads();
        }
        const unsigned below = (1u << lane) - 1u;
        for (int base = lo; base < hi; base += 32) {
            const int z = base + lane;
            const int j = z < hi ? nbr[z] - a0 : -1;
            const unsigned same = __match_any_sync(0xffffffffu, j);
            int dst = 0;
            if (j >= 0) dst = h[j] + __popc(same & below);
            __syncwarp();
            if (j >= 0) {
                col_perm[dst] = z;
                if ((same >> lane) == 1u) h[j] += __popc(same);  // the group's last lane moves the column on
            }
            __syncwarp();
        }
    }
    __syncthreads();
    if (t == 0) frame_flag[b] = 0;  // the next rebuild starts from no flag
}

template <bool FILL>
int slots_walk(int pos_dtype, int64_t n, int64_t B, const int32_t* frame_ptr, const void* pos, const void* cell, const void* inv,
               const int32_t* pbc, const int32_t* nimg, double r_max, const int32_t* frame_flag, int32_t* counts,
               const int32_t* row_ptr, double pad, int32_t* ctr, int32_t* nbr, void* shift, void* pos_ref, void* stream) {
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    AB2_CHECK_ARG(B >= 1 && frame_ptr && pos && cell && inv && pbc && nimg && frame_flag, "null pointer or no frame");
    AB2_CHECK_ARG(r_max > 0, "r_max must be positive");
    AB2_CHECK_ARG(FILL ? (row_ptr && ctr && nbr && shift && pos_ref) : (counts != nullptr), "null output pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = ab2_blocks(n, NLF_WARPS);
    if (pos_dtype == AB2_F64)
        nlf_walk_kernel<double, FILL, true><<<grid, NLF_WARPS * 32, 0, st>>>(
            n, B, frame_ptr, (const double*)pos, (const double*)cell, (const double*)inv, pbc, nimg, r_max, counts, row_ptr, nbr,
            (double*)shift, frame_flag, ctr, (double*)pos_ref, pad);
    else
        nlf_walk_kernel<float, FILL, true><<<grid, NLF_WARPS * 32, 0, st>>>(
            n, B, frame_ptr, (const float*)pos, (const float*)cell, (const float*)inv, pbc, nimg, r_max, counts, row_ptr, nbr,
            (float*)shift, frame_flag, ctr, (float*)pos_ref, pad);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

size_t slots_transpose_smem(int max_frame_atoms) { return (size_t)(SLOT_T_WARPS + 1) * (size_t)max_frame_atoms * sizeof(int32_t); }

}  // namespace

extern "C" int ab2_slots_check(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos, const void* pos_ref,
                               double half_skin, int32_t* frame_flag, void* stream) {
    if (n == 0) return 0;
    AB2_CHECK_ARG(pos_dtype == AB2_F64 || pos_dtype == AB2_F32, "positions must be fp64 or fp32");
    AB2_CHECK_ARG(n_frames >= 1 && frame_ptr && pos && pos_ref && frame_flag, "null pointer or no frame");
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = ab2_blocks(n, SLOT_CHECK_THREADS);
    if (pos_dtype == AB2_F64)
        slots_check_kernel<double><<<grid, SLOT_CHECK_THREADS, 0, st>>>(n, n_frames, frame_ptr, (const double*)pos, (const double*)pos_ref,
                                                                         half_skin, frame_flag);
    else
        slots_check_kernel<float><<<grid, SLOT_CHECK_THREADS, 0, st>>>(n, n_frames, frame_ptr, (const float*)pos, (const float*)pos_ref,
                                                                        (float)half_skin, frame_flag);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_slots_count(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos, const void* cell,
                               const void* inv_cell, const int32_t* pbc, const int32_t* nimg, double r_max, const int32_t* frame_flag,
                               int32_t* counts, void* stream) {
    return slots_walk<false>(pos_dtype, n, n_frames, frame_ptr, pos, cell, inv_cell, pbc, nimg, r_max, frame_flag, counts, nullptr, 0.0,
                             nullptr, nullptr, nullptr, nullptr, stream);
}

extern "C" int ab2_slots_place(int64_t n_frames, const int32_t* frame_ptr, const int32_t* slot_ptr, const int32_t* counts,
                               int32_t* frame_flag, int32_t* row_ptr, int32_t* overflow, int32_t* rebuilds, void* stream) {
    AB2_CHECK_ARG(n_frames >= 1 && frame_ptr && slot_ptr && counts && frame_flag && row_ptr && overflow && rebuilds, "null pointer or no frame");
    slots_place_kernel<<<(unsigned)n_frames, SLOT_PLACE_THREADS, 0, (cudaStream_t)stream>>>(frame_ptr, slot_ptr, counts, frame_flag, row_ptr,
                                                                                             overflow, rebuilds);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

extern "C" int ab2_slots_fill(int pos_dtype, int64_t n, int64_t n_frames, const int32_t* frame_ptr, const void* pos, const void* cell,
                              const void* inv_cell, const int32_t* pbc, const int32_t* nimg, double r_max, const int32_t* frame_flag,
                              const int32_t* row_ptr, double pad, int32_t* ctr, int32_t* nbr, void* shift, void* pos_ref, void* stream) {
    return slots_walk<true>(pos_dtype, n, n_frames, frame_ptr, pos, cell, inv_cell, pbc, nimg, r_max, frame_flag, nullptr, row_ptr, pad,
                            ctr, nbr, shift, pos_ref, stream);
}

extern "C" int ab2_slots_transpose(int64_t n_frames, int max_frame_atoms, const int32_t* frame_ptr, const int32_t* slot_ptr,
                                   const int32_t* nbr, int32_t* frame_flag, int32_t* col_ptr, int32_t* col_perm, void* stream) {
    AB2_CHECK_ARG(n_frames >= 1 && frame_ptr && slot_ptr && frame_flag && col_ptr && col_perm, "null pointer or no frame");
    AB2_CHECK_ARG(max_frame_atoms >= 0 && max_frame_atoms <= AB2_FRAMES_MAX_ATOMS, "max_frame_atoms outside [0, AB2_FRAMES_MAX_ATOMS]");
    const size_t smem = slots_transpose_smem(max_frame_atoms);
    // the largest histograms need more than the default 48 KB: allowed once per device, on the first (uncaptured) build
    static unsigned long long raised = 0;
    int dev = 0;
    AB2_CUDA_CALL(cudaGetDevice(&dev));
    if (dev < 64 && !((raised >> dev) & 1ull)) {
        AB2_CUDA_CALL(cudaFuncSetAttribute(slots_transpose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                           (int)slots_transpose_smem(AB2_FRAMES_MAX_ATOMS)));
        raised |= 1ull << dev;
    }
    slots_transpose_kernel<<<(unsigned)n_frames, SLOT_T_WARPS * 32, smem, (cudaStream_t)stream>>>(frame_ptr, slot_ptr, nbr, frame_flag,
                                                                                                   col_ptr, col_perm);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

// Ghost-atom halo exchange over NVLink peer memory -- no NCCL call on the per-step path.
//
// Spatial decomposition (SURVEY section 8e): per force evaluation a rank sends the positions of its boundary atoms to
// the two neighbouring slabs (forward halo), receives the gradients accumulated on its ghosts' owners' behalf back
// (reverse halo), and all ranks sum one scalar energy.  Messages are tens of KB, so the cost is latency: through
// torch.distributed / NCCL point-to-point the three exchanges add pack / unpack torch kernels and NCCL kernels to every
// step inside the CUDA graph.  Here every rank owns a small MAILBOX allocation that its peers map
// through CUDA IPC; the sender's kernel gathers the rows and STORES them straight into the receiver's mailbox over
// NVLink, then publishes the step number with a system-scope release store; the receiver's kernel spins on that flag
// (acquire) and unpacks.  Everything is ordinary kernels, so the whole step -- halo included -- stays one CUDA graph.
//
// Mailbox layout (double buffered by the parity of the step number: a sender can be at most one step ahead of a peer
// -- its next step needs that peer's data of the current one -- so the slot it overwrites was consumed a step ago):
//   [parity][side] ghost positions    (3 * max_rows doubles)   side 0: written by my LEFT neighbour, 1: by my RIGHT one
//   [parity][side] boundary gradients (3 * max_rows doubles)
//   [parity][rank] energies (double)
//   flags (uint32 step numbers): pos[parity][side], grad[parity][side], energy[parity][rank]; then an error word
//
// Extended mailbox (ab2_p2p_mailbox_bytes_ex with AB2_P2P_EXT_VIRIAL): the base layout above, unchanged (so the error
// word stays where ab2_p2p_error looks), then, from the next 256-byte boundary
//   [parity][side] reverse rows of width 12 (3 gradient + 9 per-atom virial values, fp64; 12 * max_rows doubles)
//   [parity][rank] a vector of up to AB2_P2P_VEC_MAX doubles (energy, virial, heat current)
//   flags: wrows[parity][side], vec[parity][rank]
#include <type_traits>

#include "common.cuh"

namespace {

struct MailboxLayout {
    int max_rows, world;
    __host__ __device__ size_t rows_bytes() const { return (size_t)3 * max_rows * 8; }
    __host__ __device__ size_t pos_off(int par, int side) const { return (size_t)(par * 2 + side) * rows_bytes(); }
    __host__ __device__ size_t grad_off(int par, int side) const { return (size_t)(4 + par * 2 + side) * rows_bytes(); }
    __host__ __device__ size_t e_off(int par) const { return 8 * rows_bytes() + (size_t)par * world * 8; }
    __host__ __device__ size_t flag_off() const { return 8 * rows_bytes() + (size_t)2 * world * 8; }
    __host__ __device__ int pos_flag(int par, int side) const { return par * 2 + side; }
    __host__ __device__ int grad_flag(int par, int side) const { return 4 + par * 2 + side; }
    __host__ __device__ int e_flag(int par, int rank) const { return 8 + par * world + rank; }
    __host__ __device__ int err_word() const { return 8 + 2 * world; }
    __host__ __device__ size_t bytes() const { return flag_off() + (size_t)(err_word() + 1) * 4 + 64; }
};

struct ExtLayout {
    MailboxLayout B;
    __host__ __device__ size_t base() const { return (B.bytes() + 255) & ~(size_t)255; }
    __host__ __device__ size_t wrows_bytes() const { return (size_t)12 * B.max_rows * 8; }
    __host__ __device__ size_t wrows_off(int par, int side) const { return base() + (size_t)(par * 2 + side) * wrows_bytes(); }
    __host__ __device__ size_t vec_off(int par, int rank) const {
        return base() + 4 * wrows_bytes() + ((size_t)par * B.world + rank) * AB2_P2P_VEC_MAX * 8;
    }
    __host__ __device__ size_t flag_off() const { return base() + 4 * wrows_bytes() + (size_t)2 * B.world * AB2_P2P_VEC_MAX * 8; }
    __host__ __device__ int wrows_flag(int par, int side) const { return par * 2 + side; }
    __host__ __device__ int vec_flag(int par, int rank) const { return 4 + par * B.world + rank; }
    __host__ __device__ size_t bytes() const { return flag_off() + (size_t)(4 + 2 * B.world) * 4 + 64; }
    // the one error word of the mailbox, in the base layout
    __host__ __device__ uint32_t* err(uint8_t* mailbox) const { return reinterpret_cast<uint32_t*>(mailbox + B.flag_off()) + B.err_word(); }
};

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// spin until *flag >= want (step numbers only grow); bounded so that a protocol bug cannot hang the GPU
__device__ __forceinline__ bool wait_flag(const uint32_t* flag, uint32_t want, uint32_t* err) {
    const long long t0 = clock64();
    while ((int32_t)(ld_acquire_sys(flag) - want) < 0) {
        if (clock64() - t0 > 4000000000LL) {  // ~2 s
            atomicExch(err, 1u);
            return false;
        }
        __nanosleep(64);
    }
    return true;
}

// step counter: the first kernel of every step bumps it; all later kernels of the step read it
__global__ void p2p_begin_kernel(uint32_t* step) { *step += 1; }

// kind 0: positions (x shifted), 1: gradients.  rows src[idx[i]] (or src[i]) -> the PEER's mailbox slot `side` of the
// current step's parity, then publish the step number (last block, after a system-scope fence).
// VEC = true (ab2_p2p_push_rows_v): the shift is a vector (a lattice row of a triclinic cell), added to all three components
struct Shift3 {
    double v[3];
};

template <typename TSrc, bool VEC>
__global__ void __launch_bounds__(256) p2p_push_rows_kernel(MailboxLayout L, int kind, int side, const TSrc* __restrict__ src,
                                                            const int64_t* __restrict__ idx, int n, std::conditional_t<VEC, Shift3, double> shift_x,
                                                            uint8_t* __restrict__ peer, const uint32_t* __restrict__ step, uint32_t* __restrict__ done_ctr) {
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    double* __restrict__ dst = reinterpret_cast<double*>(peer + (kind == 0 ? L.pos_off(par, side) : L.grad_off(par, side)));
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) {
        const int64_t r = idx ? idx[i] : i;
        if constexpr (VEC) {
            dst[3 * i + 0] = (double)src[3 * r + 0] + shift_x.v[0];
            dst[3 * i + 1] = (double)src[3 * r + 1] + shift_x.v[1];
            dst[3 * i + 2] = (double)src[3 * r + 2] + shift_x.v[2];
        } else {
            dst[3 * i + 0] = (double)src[3 * r + 0] + shift_x;
            dst[3 * i + 1] = (double)src[3 * r + 1];
            dst[3 * i + 2] = (double)src[3 * r + 2];
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t prev = atomicAdd(done_ctr, 1u);
        if (prev == gridDim.x - 1) {  // last block: every block's rows are visible system-wide
            *done_ctr = 0;
            __threadfence_system();
            uint32_t* flags = reinterpret_cast<uint32_t*>(peer + L.flag_off());
            st_release_sys(flags + (kind == 0 ? L.pos_flag(par, side) : L.grad_flag(par, side)), s);
        }
    }
}

// wait for the rows a neighbour pushed into MY mailbox this step, then unpack: dst[idx[i] or off + i] (=|+=) row i
template <typename TDst>
__global__ void __launch_bounds__(256) p2p_wait_unpack_kernel(MailboxLayout L, int kind, int side, uint8_t* __restrict__ mine,
                                                              const uint32_t* __restrict__ step, int n, TDst* __restrict__ dst,
                                                              const int64_t* __restrict__ idx, int accumulate) {
    __shared__ int ok;
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    uint32_t* flags = reinterpret_cast<uint32_t*>(mine + L.flag_off());
    if (threadIdx.x == 0) ok = wait_flag(flags + (kind == 0 ? L.pos_flag(par, side) : L.grad_flag(par, side)), s, flags + L.err_word()) ? 1 : 0;
    __syncthreads();
    if (!ok) return;
    const double* __restrict__ box = reinterpret_cast<const double*>(mine + (kind == 0 ? L.pos_off(par, side) : L.grad_off(par, side)));
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i < n) {
        const int64_t r = idx ? idx[i] : i;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const double v = box[3 * i + a];
            if (accumulate) dst[3 * r + a] += (TDst)v;
            else dst[3 * r + a] = (TDst)v;
        }
    }
}

__global__ void p2p_push_energy_kernel(MailboxLayout L, const double* __restrict__ e_local, int rank, uint8_t* const* __restrict__ peers,
                                       const uint32_t* __restrict__ step) {
    const int r = threadIdx.x;
    if (r >= L.world) return;
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    uint8_t* peer = peers[r];
    reinterpret_cast<double*>(peer + L.e_off(par))[rank] = *e_local;
    __threadfence_system();
    st_release_sys(reinterpret_cast<uint32_t*>(peer + L.flag_off()) + L.e_flag(par, rank), s);
}

__global__ void p2p_sum_energy_kernel(MailboxLayout L, uint8_t* __restrict__ mine, const uint32_t* __restrict__ step, double* __restrict__ out) {
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    uint32_t* flags = reinterpret_cast<uint32_t*>(mine + L.flag_off());
    const double* e = reinterpret_cast<const double*>(mine + L.e_off(par));
    double tot = 0.0;
    for (int r = 0; r < L.world; ++r) {  // fixed order: bitwise identical total on every rank
        if (!wait_flag(flags + L.e_flag(par, r), s, flags + L.err_word())) return;
        tot += e[r];
    }
    *out = tot;
}

// Reverse rows of width 12: gradient row i (g[3i..3i+2]) and per-atom virial row i (W[9i..9i+8]) -> the PEER's wrows
// slot `side`, one element per thread so that the stores over NVLink are contiguous; then the flag, as above.
template <typename TSrc>
__global__ void __launch_bounds__(256) p2p_push_wrows_kernel(ExtLayout L, int side, const TSrc* __restrict__ g, const TSrc* __restrict__ W,
                                                             int n, uint8_t* __restrict__ peer, const uint32_t* __restrict__ step,
                                                             uint32_t* __restrict__ done_ctr) {
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    double* __restrict__ dst = reinterpret_cast<double*>(peer + L.wrows_off(par, side));
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e < (int64_t)12 * n) {
        const int64_t i = e / 12;
        const int c = (int)(e - 12 * i);
        dst[e] = c < 3 ? (double)g[3 * i + c] : (double)W[9 * i + (c - 3)];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t prev = atomicAdd(done_ctr, 1u);
        if (prev == gridDim.x - 1) {
            *done_ctr = 0;
            __threadfence_system();
            uint32_t* flags = reinterpret_cast<uint32_t*>(peer + L.flag_off());
            st_release_sys(flags + L.wrows_flag(par, side), s);
        }
    }
}

// wait for this step's width-12 rows in MY mailbox slot `side`, then g_dst[idx[i]] += gradient row i and
// W_dst[idx[i]] += virial row i (idx unique within one call, so one launch adds both without atomics)
template <typename TDst>
__global__ void __launch_bounds__(256) p2p_wait_unpack_wrows_kernel(ExtLayout L, int side, uint8_t* __restrict__ mine, const uint32_t* __restrict__ step,
                                                                    int n, TDst* __restrict__ g_dst, TDst* __restrict__ W_dst,
                                                                    const int64_t* __restrict__ idx) {
    __shared__ int ok;
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    const uint32_t* flags = reinterpret_cast<const uint32_t*>(mine + L.flag_off());
    if (threadIdx.x == 0) ok = wait_flag(flags + L.wrows_flag(par, side), s, L.err(mine)) ? 1 : 0;
    __syncthreads();
    if (!ok) return;
    const double* __restrict__ box = reinterpret_cast<const double*>(mine + L.wrows_off(par, side));
    const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (e < (int64_t)12 * n) {
        const int64_t i = e / 12;
        const int c = (int)(e - 12 * i);
        const int64_t r = idx ? idx[i] : i;
        const double v = box[e];
        if (c < 3) g_dst[3 * r + c] += (TDst)v;
        else W_dst[9 * r + (c - 3)] += (TDst)v;
    }
}

// thread r stores my n_values doubles into rank r's vec slot [parity][my rank], then publishes the step number
__global__ void p2p_push_vec_kernel(ExtLayout L, const double* __restrict__ v_local, int n_values, int rank, uint8_t* const* __restrict__ peers,
                                    const uint32_t* __restrict__ step) {
    const int r = threadIdx.x;
    if (r >= L.B.world) return;
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    uint8_t* peer = peers[r];
    double* dst = reinterpret_cast<double*>(peer + L.vec_off(par, rank));
    for (int k = 0; k < n_values; ++k) dst[k] = v_local[k];
    __threadfence_system();
    st_release_sys(reinterpret_cast<uint32_t*>(peer + L.flag_off()) + L.vec_flag(par, rank), s);
}

// thread 0 waits for every rank's vector; then thread k sums component k over the ranks in rank order (bitwise
// identical on every rank, and component 0 bitwise equal to what p2p_sum_energy_kernel gives for the same values)
__global__ void p2p_sum_vec_kernel(ExtLayout L, uint8_t* __restrict__ mine, const uint32_t* __restrict__ step, int n_values, double* __restrict__ out) {
    __shared__ int ok;
    const uint32_t s = *step;
    const int par = (int)(s & 1u);
    const uint32_t* flags = reinterpret_cast<const uint32_t*>(mine + L.flag_off());
    if (threadIdx.x == 0) {
        ok = 1;
        for (int r = 0; r < L.B.world && ok; ++r) ok = wait_flag(flags + L.vec_flag(par, r), s, L.err(mine)) ? 1 : 0;
    }
    __syncthreads();
    if (!ok) return;
    const int k = threadIdx.x;
    if (k >= n_values) return;
    double tot = 0.0;
    for (int r = 0; r < L.B.world; ++r) tot += reinterpret_cast<const double*>(mine + L.vec_off(par, r))[k];
    out[k] = tot;
}

}  // namespace

// ---- host API (C ABI) -----------------------------------------------------------------------------------------
extern "C" int64_t ab2_p2p_mailbox_bytes(int max_rows, int world) {
    MailboxLayout L{max_rows, world};
    return (int64_t)L.bytes();
}
extern "C" int ab2_p2p_alloc(int64_t bytes, void** ptr) {
    AB2_CHECK_ARG(ptr && bytes > 0, "bad arguments");
    AB2_CUDA_CALL(cudaMalloc(ptr, (size_t)bytes));
    AB2_CUDA_CALL(cudaMemset(*ptr, 0, (size_t)bytes));
    AB2_CUDA_CALL(cudaDeviceSynchronize());
    return 0;
}
extern "C" int ab2_p2p_free(void* ptr) {
    if (ptr) AB2_CUDA_CALL(cudaFree(ptr));
    return 0;
}
extern "C" int ab2_p2p_get_handle(void* ptr, void* handle64_host) {
    AB2_CHECK_ARG(ptr && handle64_host, "null pointer");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    AB2_CUDA_CALL(cudaIpcGetMemHandle((cudaIpcMemHandle_t*)handle64_host, ptr));
    return 0;
}
extern "C" int ab2_p2p_open_handle(const void* handle64_host, void** ptr) {
    AB2_CHECK_ARG(ptr && handle64_host, "null pointer");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64_host, 64);
    AB2_CUDA_CALL(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}
extern "C" int ab2_p2p_close_handle(void* ptr) {
    if (ptr) AB2_CUDA_CALL(cudaIpcCloseMemHandle(ptr));
    return 0;
}
/* error word of my mailbox (1 = a wait timed out), copied to the host (synchronises the stream) */
extern "C" int ab2_p2p_error(void* my_mailbox, int max_rows, int world, void* stream) {
    MailboxLayout L{max_rows, world};
    uint32_t v = 0;
    AB2_CUDA_CALL(cudaMemcpyAsync(&v, (uint8_t*)my_mailbox + L.flag_off() + (size_t)L.err_word() * 4, 4, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    AB2_CUDA_CALL(cudaStreamSynchronize((cudaStream_t)stream));
    return (int)v;
}

extern "C" int ab2_p2p_begin(void* step_counter, void* stream) {
    AB2_CHECK_ARG(step_counter, "null pointer");
    p2p_begin_kernel<<<1, 1, 0, (cudaStream_t)stream>>>((uint32_t*)step_counter);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* Push n rows of src ([.,3] fp64 / fp32; rows idx[i], or 0..n-1 if idx is null) into the PEER's mailbox.  kind 0 =
 * positions (x shifted by shift_x), 1 = gradients; side = the slot of the peer's mailbox (0: "written by its left
 * neighbour", 1: "by its right neighbour").  done_counter: one zeroed uint32 of scratch per concurrent push. */
extern "C" int ab2_p2p_push_rows(int src_dtype, int kind, int side, const void* src, const int64_t* idx, int n, double shift_x, void* peer_mailbox,
                                 int max_rows, int world, const void* step_counter, void* done_counter, void* stream) {
    AB2_CHECK_ARG(src && peer_mailbox && step_counter && done_counter && n >= 0 && n <= max_rows, "bad arguments");
    AB2_CHECK_ARG(src_dtype == AB2_F64 || src_dtype == AB2_F32, "rows must be fp64 or fp32");
    MailboxLayout L{max_rows, world};
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = n > 0 ? ab2_blocks(n, 256) : 1;
    if (src_dtype == AB2_F64)
        p2p_push_rows_kernel<double, false><<<grid, 256, 0, st>>>(L, kind, side, (const double*)src, idx, n, shift_x, (uint8_t*)peer_mailbox,
                                                          (const uint32_t*)step_counter, (uint32_t*)done_counter);
    else
        p2p_push_rows_kernel<float, false><<<grid, 256, 0, st>>>(L, kind, side, (const float*)src, idx, n, shift_x, (uint8_t*)peer_mailbox,
                                                         (const uint32_t*)step_counter, (uint32_t*)done_counter);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* ab2_p2p_push_rows with the shift (shift_x, shift_y, shift_z) added to every component: a ghost crossing the periodic
 * face of lattice row 0 of a triclinic cell moves by that row.  The shift is passed by value (graph-capturable). */
extern "C" int ab2_p2p_push_rows_v(int src_dtype, int kind, int side, const void* src, const int64_t* idx, int n, double shift_x, double shift_y,
                                   double shift_z, void* peer_mailbox, int max_rows, int world, const void* step_counter, void* done_counter,
                                   void* stream) {
    AB2_CHECK_ARG(src && peer_mailbox && step_counter && done_counter && n >= 0 && n <= max_rows, "bad arguments");
    AB2_CHECK_ARG(src_dtype == AB2_F64 || src_dtype == AB2_F32, "rows must be fp64 or fp32");
    MailboxLayout L{max_rows, world};
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = n > 0 ? ab2_blocks(n, 256) : 1;
    const Shift3 sh{{shift_x, shift_y, shift_z}};
    if (src_dtype == AB2_F64)
        p2p_push_rows_kernel<double, true><<<grid, 256, 0, st>>>(L, kind, side, (const double*)src, idx, n, sh, (uint8_t*)peer_mailbox,
                                                                (const uint32_t*)step_counter, (uint32_t*)done_counter);
    else
        p2p_push_rows_kernel<float, true><<<grid, 256, 0, st>>>(L, kind, side, (const float*)src, idx, n, sh, (uint8_t*)peer_mailbox,
                                                               (const uint32_t*)step_counter, (uint32_t*)done_counter);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* Wait for this step's rows in MY mailbox slot (kind, side) and unpack them: dst[idx[i] or i] = / += row i. */
extern "C" int ab2_p2p_wait_unpack(int dst_dtype, int kind, int side, void* my_mailbox, int max_rows, int world, const void* step_counter, int n,
                                   void* dst, const int64_t* idx, int accumulate, void* stream) {
    AB2_CHECK_ARG(my_mailbox && step_counter && dst && n >= 0 && n <= max_rows, "bad arguments");
    AB2_CHECK_ARG(dst_dtype == AB2_F64 || dst_dtype == AB2_F32, "rows must be fp64 or fp32");
    MailboxLayout L{max_rows, world};
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = n > 0 ? ab2_blocks(n, 256) : 1;
    if (dst_dtype == AB2_F64)
        p2p_wait_unpack_kernel<double><<<grid, 256, 0, st>>>(L, kind, side, (uint8_t*)my_mailbox, (const uint32_t*)step_counter, n, (double*)dst, idx, accumulate);
    else
        p2p_wait_unpack_kernel<float><<<grid, 256, 0, st>>>(L, kind, side, (uint8_t*)my_mailbox, (const uint32_t*)step_counter, n, (float*)dst, idx, accumulate);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* All-reduce of one double without NCCL: push my value into every rank's mailbox, then sum the world's values in rank
 * order.  peers_dev: device array of world mailbox pointers (own mailbox at index rank). */
extern "C" int ab2_p2p_allreduce_energy(const void* e_local, int rank, int world, int max_rows, void* const* peers_dev, void* my_mailbox,
                                        const void* step_counter, void* e_total, void* stream) {
    AB2_CHECK_ARG(e_local && peers_dev && my_mailbox && step_counter && e_total && world >= 1 && world <= 64, "bad arguments");
    MailboxLayout L{max_rows, world};
    cudaStream_t st = (cudaStream_t)stream;
    p2p_push_energy_kernel<<<1, 64, 0, st>>>(L, (const double*)e_local, rank, (uint8_t* const*)peers_dev, (const uint32_t*)step_counter);
    p2p_sum_energy_kernel<<<1, 1, 0, st>>>(L, (uint8_t*)my_mailbox, (const uint32_t*)step_counter, (double*)e_total);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* Size of a mailbox with the optional sections of `flags` (0: exactly ab2_p2p_mailbox_bytes; AB2_P2P_EXT_VIRIAL: the
 * width-12 reverse rows and the vector all-reduce).  -1 for unknown flag bits. */
extern "C" int64_t ab2_p2p_mailbox_bytes_ex(int max_rows, int world, int flags) {
    if (flags & ~AB2_P2P_EXT_VIRIAL) return -1;
    MailboxLayout B{max_rows, world};
    if (!flags) return (int64_t)B.bytes();
    return (int64_t)ExtLayout{B}.bytes();
}

/* Push n reverse rows of width 12 -- gradient rows g[i][3] and per-atom virial rows W[i][3][3], i < n, both fp64 or both
 * fp32 -- into the PEER's (extended) mailbox slot `side`. */
extern "C" int ab2_p2p_push_rows_w(int src_dtype, int side, const void* g_src, const void* W_src, int n, void* peer_mailbox, int max_rows,
                                   int world, const void* step_counter, void* done_counter, void* stream) {
    AB2_CHECK_ARG(g_src && W_src && peer_mailbox && step_counter && done_counter && n >= 0 && n <= max_rows && (side == 0 || side == 1),
                  "bad arguments");
    AB2_CHECK_ARG(src_dtype == AB2_F64 || src_dtype == AB2_F32, "rows must be fp64 or fp32");
    ExtLayout L{MailboxLayout{max_rows, world}};
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = n > 0 ? ab2_blocks((int64_t)12 * n, 256) : 1;
    if (src_dtype == AB2_F64)
        p2p_push_wrows_kernel<double><<<grid, 256, 0, st>>>(L, side, (const double*)g_src, (const double*)W_src, n, (uint8_t*)peer_mailbox,
                                                           (const uint32_t*)step_counter, (uint32_t*)done_counter);
    else
        p2p_push_wrows_kernel<float><<<grid, 256, 0, st>>>(L, side, (const float*)g_src, (const float*)W_src, n, (uint8_t*)peer_mailbox,
                                                          (const uint32_t*)step_counter, (uint32_t*)done_counter);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* Wait for this step's width-12 rows in MY (extended) mailbox slot `side` and add them: g_dst[idx[i]] += gradient row i,
 * W_dst[idx[i]] += virial row i (idx null: row i). */
extern "C" int ab2_p2p_wait_unpack_w(int dst_dtype, int side, void* my_mailbox, int max_rows, int world, const void* step_counter, int n,
                                     void* g_dst, void* W_dst, const int64_t* idx, void* stream) {
    AB2_CHECK_ARG(my_mailbox && step_counter && g_dst && W_dst && n >= 0 && n <= max_rows && (side == 0 || side == 1), "bad arguments");
    AB2_CHECK_ARG(dst_dtype == AB2_F64 || dst_dtype == AB2_F32, "rows must be fp64 or fp32");
    ExtLayout L{MailboxLayout{max_rows, world}};
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned grid = n > 0 ? ab2_blocks((int64_t)12 * n, 256) : 1;
    if (dst_dtype == AB2_F64)
        p2p_wait_unpack_wrows_kernel<double><<<grid, 256, 0, st>>>(L, side, (uint8_t*)my_mailbox, (const uint32_t*)step_counter, n, (double*)g_dst,
                                                                  (double*)W_dst, idx);
    else
        p2p_wait_unpack_wrows_kernel<float><<<grid, 256, 0, st>>>(L, side, (uint8_t*)my_mailbox, (const uint32_t*)step_counter, n, (float*)g_dst,
                                                                 (float*)W_dst, idx);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

/* All-reduce of n_values <= AB2_P2P_VEC_MAX doubles through the extended mailboxes: the ab2_p2p_allreduce_energy protocol
 * for a vector; v_total[k] = sum over ranks in rank order of v_local[k], bitwise identical on every rank. */
extern "C" int ab2_p2p_allreduce_vec(const void* v_local, int n_values, int rank, int world, int max_rows, void* const* peers_dev,
                                     void* my_mailbox, const void* step_counter, void* v_total, void* stream) {
    AB2_CHECK_ARG(v_local && peers_dev && my_mailbox && step_counter && v_total && world >= 1 && world <= 64 && rank >= 0 && rank < world,
                  "bad arguments");
    AB2_CHECK_ARG(n_values >= 1 && n_values <= AB2_P2P_VEC_MAX, "n_values must be in [1, 16]");
    ExtLayout L{MailboxLayout{max_rows, world}};
    cudaStream_t st = (cudaStream_t)stream;
    p2p_push_vec_kernel<<<1, 64, 0, st>>>(L, (const double*)v_local, n_values, rank, (uint8_t* const*)peers_dev, (const uint32_t*)step_counter);
    p2p_sum_vec_kernel<<<1, 32, 0, st>>>(L, (uint8_t*)my_mailbox, (const uint32_t*)step_counter, n_values, (double*)v_total);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

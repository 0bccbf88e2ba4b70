// fp64 tensor product for the l_max = 3 layer shapes (BASELINE configs[4]: 16 x 16 -> 31, 31 x 16 -> 16, 16 x 16 -> 1) with the
// coupling-table STRUCTURE baked at compile time.
//
// Reference semantics: Contracter._contract (allegro/nn/_strided/_contract.py:213-251) after the scatter/gather of :199-205,
// and its two backward products (_flashallegro.py:347-360), on centre-sorted edges and the component-major layout; layer 0
// with V0 = Y (x) w0 formed on the fly (tensorembed.py:95).
//
// Why.  The shape-generic kernels (tp.cu) walk the run-time table per (edge, channel) with dynamically indexed per-thread
// arrays -> local memory, three index loads and two global loads per entry, which makes them the larger part of the c5
// step.  The table's (i, j, k) structure is fixed by the selection rules (tools/gen_tp_tables.py emits it
// as constexpr), only cgw[nnz][u] is data.  With the structure baked the 611-entry contraction is straight-line DFMAs on
// REGISTERS (<= 63 live doubles: the backward runs its two products as two launches -- in one kernel the compiler parks
// ~5 KB per thread in local memory between the passes), the 32-channel slice of
// cgw a CTA needs sits in shared memory (156 KB, read once per CTA), and every global access is a coalesced 256-byte row.
// One thread per (edge, channel), lane = channel, a warp per edge; persistent grid (#SMs x channel chunks).
//
// The kernel checks the run-time table against the baked structure (constant memory) and tells the caller's fallback through
// a device flag: 1 = "done here", 0 = "not my table" -> the shape-generic kernel launched right behind it does the work.
#include "common.cuh"
#include "tp_fast.cuh"
#include "tp_tables_generated.cuh"

int g_ab2_opt_tp_baked64 = 1;  // 1: baked fp64 kernels for the l_max = 3 shapes, 0: shape-generic kernels only

namespace {

constexpr int THREADS = 384, NW = THREADS / 32;

template <typename TAB>
struct Packed {
    uint32_t v[TAB::NNZ];
};
template <typename TAB>
constexpr Packed<TAB> make_packed() {
    Packed<TAB> t{};
    for (int n = 0; n < TAB::NNZ; ++n) t.v[n] = (uint32_t)TAB::I(n) | ((uint32_t)TAB::J(n) << 8) | ((uint32_t)TAB::K(n) << 16);
    return t;
}
__constant__ Packed<Tab16x16x31> c_tab_a = make_packed<Tab16x16x31>();
__constant__ Packed<Tab31x16x16> c_tab_b = make_packed<Tab31x16x16>();
__constant__ Packed<Tab16x16x1> c_tab_c = make_packed<Tab16x16x1>();
template <typename TAB>
__device__ __forceinline__ const uint32_t* packed_tab();
template <>
__device__ __forceinline__ const uint32_t* packed_tab<Tab16x16x31>() { return c_tab_a.v; }
template <>
__device__ __forceinline__ const uint32_t* packed_tab<Tab31x16x16>() { return c_tab_b.v; }
template <>
__device__ __forceinline__ const uint32_t* packed_tab<Tab16x16x1>() { return c_tab_c.v; }

struct Params64 {
    int64_t E;
    int U;
    const int32_t* tab;
    const double* cgw;
    const int32_t* ctr;
    const double* gamma;
    const double* Vin;
    const double* Y;
    const double* w0;
    int64_t w0_ld;
    double* Vout;
    const double* gVout;
    double* gVin;
    double* gw0;
    int64_t gw0_ld;
    double* gY;
    double* ggamma;
    int* flag;
};

template <typename TAB, int MODE, bool IMPLICIT>
__global__ void __launch_bounds__(THREADS, 1) tp_baked64_kernel(const Params64 p) {
    constexpr int NNZ = TAB::NNZ, D_IN = TAB::D_IN, D = TAB::D_ENV, D_OUT = TAB::D_OUT;
    extern __shared__ double s_cgw[];  // [NNZ][32]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    {
        const uint32_t* want = packed_tab<TAB>();
        int ok = 1;
        for (int n = tid; n < NNZ; n += THREADS)
            if (((uint32_t)p.tab[3 * n] | ((uint32_t)p.tab[3 * n + 1] << 8) | ((uint32_t)p.tab[3 * n + 2] << 16)) != want[n]) ok = 0;
        ok = __syncthreads_and(ok);
        if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0) *p.flag = ok;
        if (!ok) return;
    }
    const int U = p.U, u0 = blockIdx.y * 32, u = u0 + lane;
    for (int e = tid; e < NNZ * 32; e += THREADS) s_cgw[e] = p.cgw[(int64_t)(e >> 5) * U + u0 + (e & 31)];
    __syncthreads();
    const double* __restrict__ cg = s_cgw + lane;
    for (int64_t z = (int64_t)blockIdx.x * NW + warp; z < p.E; z += (int64_t)gridDim.x * NW) {
        const int64_t c = p.ctr[z];
        [[maybe_unused]] double g[D];
        if constexpr (MODE != 2) {
#pragma unroll
            for (int j = 0; j < D; ++j) g[j] = p.gamma[(c * D + j) * U + u];
        }
        if constexpr (MODE == 0) {
            double vin[D_IN];
            if constexpr (IMPLICIT) {
#pragma unroll
                for (int i = 0; i < D_IN; ++i) vin[i] = p.Y[z * D_IN + i] * p.w0[z * p.w0_ld + sh_l_of(i) * U + u];
            } else {
#pragma unroll
                for (int i = 0; i < D_IN; ++i) vin[i] = p.Vin[(z * D_IN + i) * U + u];
            }
            double out[D_OUT];
#pragma unroll
            for (int k = 0; k < D_OUT; ++k) out[k] = 0.0;
#pragma unroll
            for (int n = 0; n < NNZ; ++n) {
                out[TAB::K(n)] = fma(cg[n * 32] * vin[TAB::I(n)], g[TAB::J(n)], out[TAB::K(n)]);
                if ((n & 15) == 15) asm volatile("" ::: "memory");  // keep the scheduler from hoisting all 611 shared-memory reads (spills)
            }
#pragma unroll
            for (int k = 0; k < D_OUT; ++k) p.Vout[(z * D_OUT + k) * U + u] = out[k];
        } else {
            double gout[D_OUT];
#pragma unroll
            for (int k = 0; k < D_OUT; ++k) gout[k] = p.gVout[(z * D_OUT + k) * U + u];
            if constexpr (MODE == 1) {   // pass A: gradient w.r.t. the input features
                double gin[D_IN];
#pragma unroll
                for (int i = 0; i < D_IN; ++i) gin[i] = 0.0;
#pragma unroll
                for (int n = 0; n < NNZ; ++n) {
                    gin[TAB::I(n)] = fma(cg[n * 32] * gout[TAB::K(n)], g[TAB::J(n)], gin[TAB::I(n)]);
                    if ((n & 15) == 15) asm volatile("" ::: "memory");
                }
                if constexpr (IMPLICIT) {
                    // Vin[i] = Y[i] w0[l(i)]:  gw0[l] = sum_{i in l} Y[i] gin[i];  gY[i] += sum_u w0[l(i)][u] gin[i]
#pragma unroll
                    for (int l = 0; l * l < D_IN; ++l) {
                        const double wl = p.w0[z * p.w0_ld + l * U + u];
                        double s = 0.0;
#pragma unroll
                        for (int i = l * l; i < (l + 1) * (l + 1); ++i) {
                            const double yi = p.Y[z * D_IN + i];
                            s = fma(yi, gin[i], s);
                            const double t = warp_sum(wl * gin[i]);
                            if (lane == 0) atomicAdd(&p.gY[z * D_IN + i], t);
                        }
                        p.gw0[z * p.gw0_ld + l * U + u] = s;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < D_IN; ++i) p.gVin[(z * D_IN + i) * U + u] = gin[i];
                }
            }
            if constexpr (MODE == 2) {   // pass B: gradient w.r.t. the centre's environment (accumulated over the centre's edges: atomics, like tp.cu)
                double vin[D_IN];
                if constexpr (IMPLICIT) {
#pragma unroll
                    for (int i = 0; i < D_IN; ++i) vin[i] = p.Y[z * D_IN + i] * p.w0[z * p.w0_ld + sh_l_of(i) * U + u];
                } else {
#pragma unroll
                    for (int i = 0; i < D_IN; ++i) vin[i] = p.Vin[(z * D_IN + i) * U + u];
                }
                double gg[D];
#pragma unroll
                for (int j = 0; j < D; ++j) gg[j] = 0.0;
#pragma unroll
                for (int n = 0; n < NNZ; ++n) {
                    // (cgw * vin) * gout, not (cgw * gout) * vin: the latter shares a subexpression with pass A and the compiler then
                    // parks all 611 products in local memory between the passes
                    gg[TAB::J(n)] = fma(cg[n * 32] * vin[TAB::I(n)], gout[TAB::K(n)], gg[TAB::J(n)]);
                    if ((n & 15) == 15) asm volatile("" ::: "memory");
                }
#pragma unroll
                for (int j = 0; j < D; ++j) atomicAdd(&p.ggamma[(c * D + j) * U + u], gg[j]);
            }
        }
    }
}

int* flag_buffer(cudaStream_t st) {
    static int* d_flag = nullptr;
    if (!d_flag) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {  // no allocation while capturing
            cudaGetLastError();
            return nullptr;
        }
        if (cudaMalloc(&d_flag, sizeof(int)) != cudaSuccess) {
            cudaGetLastError();
            d_flag = nullptr;
        }
    }
    return d_flag;
}

template <typename TAB, int MODE, bool IMPLICIT>
int launch64(const Params64& p, cudaStream_t st) {
    auto kern = tp_baked64_kernel<TAB, MODE, IMPLICIT>;
    const int smem = TAB::NNZ * 32 * (int)sizeof(double);
    static int num_sms = 0, ok = 0;
    if (num_sms == 0) {
        int dev = 0, max_smem = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        ok = smem <= max_smem && cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess;
        if (!ok) cudaGetLastError();
    }
    if (!ok) return -1;
    int64_t gx = num_sms;
    const int64_t need = (p.E + NW - 1) / NW;
    if (gx > need) gx = need;
    const dim3 grid((unsigned)gx, (unsigned)(p.U / 32));
    kern<<<grid, THREADS, smem, st>>>(p);
    return 0;
}

}  // namespace

// mode 0 forward, 1 backward.  Returns 0 if a kernel was launched -- *flag_out then points at a device word that the kernel
// sets to 1 when the table matched (work done) and to 0 otherwise; the caller launches its shape-generic kernel with that
// word as "skip" flag.  Returns -1 if the shape / dtype is not one of the baked ones (nothing launched).
int ab2_tp_baked64(int mode, int dtype, int64_t E, int U, int D, int d_in, int d_out, int nnz, const int32_t* tab, const void* cgw,
                   const int32_t* ctr, const void* gamma, const void* Vin, int implicit_v0, const void* Y, const void* w0, int64_t w0_ld,
                   void* Vout, const void* gVout, void* gVin, void* gw0, int64_t gw0_ld, void* gY, void* ggamma, int** flag_out,
                   cudaStream_t st) {
    if (!g_ab2_opt_tp_baked64 || dtype != AB2_F64 || D != 16 || U % 32 != 0 || E <= 0 || !ctr) return -1;
    int* flag = flag_buffer(st);
    if (!flag) return -1;
    Params64 p;
    p.E = E; p.U = U; p.tab = tab; p.cgw = (const double*)cgw; p.ctr = ctr; p.gamma = (const double*)gamma; p.Vin = (const double*)Vin;
    p.Y = (const double*)Y; p.w0 = (const double*)w0; p.w0_ld = w0_ld; p.Vout = (double*)Vout; p.gVout = (const double*)gVout;
    p.gVin = (double*)gVin; p.gw0 = (double*)gw0; p.gw0_ld = gw0_ld; p.gY = (double*)gY; p.ggamma = (double*)ggamma; p.flag = flag;
    int rc = -1;
#define AB2_B64(TAB, IMP)                                                                   \
    do {                                                                                    \
        if (mode == 0) rc = launch64<TAB, 0, IMP>(p, st);                                   \
        else {                                                                              \
            rc = launch64<TAB, 1, IMP>(p, st);                                              \
            if (rc == 0) rc = launch64<TAB, 2, IMP>(p, st);                                 \
        }                                                                                   \
    } while (0)
    if (d_in == 16 && d_out == 31 && nnz == Tab16x16x31::NNZ) {
        if (implicit_v0) AB2_B64(Tab16x16x31, true);
        else AB2_B64(Tab16x16x31, false);
    } else if (d_in == 31 && d_out == 16 && nnz == Tab31x16x16::NNZ && !implicit_v0) {
        AB2_B64(Tab31x16x16, false);
    } else if (d_in == 16 && d_out == 1 && nnz == Tab16x16x1::NNZ) {
        if (implicit_v0) AB2_B64(Tab16x16x1, true);
        else AB2_B64(Tab16x16x1, false);
    }
#undef AB2_B64
    if (rc == 0) *flag_out = flag;
    return rc;
}

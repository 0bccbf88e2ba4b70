// Committee statistics: the mean over K members of a [m][G] field and the population standard deviation of each element's
// G-vector (DP-GEN's model deviation: G = 3 gives the per-atom force deviation, G = 1 the spread of energies and of each
// virial component).
//
// One thread per element i, two passes over the members in member order, everything in fp64 with explicit round-to-nearest
// operations (no FMA contraction), each output rounded once.  So the result of element i depends on x_0[i] .. x_{K-1}[i]
// alone, never on the launch, and a torch restatement doing the same operations in the same order matches bit for bit.
//
// The K member pointers travel by value in the kernel's parameter block (a __grid_constant__ struct), so a launch needs no
// device-side table and no copy, and is captured into a CUDA graph as it is.
#include "common.cuh"

namespace {

constexpr int CM_THREADS = 256;

struct CmMembers {
    const void* p[AB2_COMMITTEE_MAX_MEMBERS];
};

template <typename T>
__global__ void __launch_bounds__(CM_THREADS) committee_moments_kernel(int K, int64_t m, int G, const __grid_constant__ CmMembers x,
                                                                       T* __restrict__ mean, T* __restrict__ dev) {
    const int64_t i = (int64_t)blockIdx.x * CM_THREADS + threadIdx.x;
    if (i >= m) return;
    const double rk = (double)K;
    double var = 0.0;
    for (int g = 0; g < G; ++g) {
        const int64_t e = i * G + g;
        // pass 1: mu = (sum_k x_k) / K, summed in member order
        double s = (double)((const T*)x.p[0])[e];
        for (int k = 1; k < K; ++k) s = __dadd_rn(s, (double)((const T*)x.p[k])[e]);
        const double mu = __ddiv_rn(s, rk);
        // pass 2: (sum_k (x_k - mu)^2) / K with the unrounded mu, in member order
        double d = __dsub_rn((double)((const T*)x.p[0])[e], mu);
        double q = __dmul_rn(d, d);
        for (int k = 1; k < K; ++k) {
            d = __dsub_rn((double)((const T*)x.p[k])[e], mu);
            q = __dadd_rn(q, __dmul_rn(d, d));
        }
        q = __ddiv_rn(q, rk);
        var = g == 0 ? q : __dadd_rn(var, q);
        mean[e] = (T)mu;
    }
    dev[i] = (T)__dsqrt_rn(var);
}

}  // namespace

extern "C" int ab2_committee_moments(int dtype, int K, int64_t m, int G, const void* const* x, void* mean, void* dev, void* stream) {
    AB2_CHECK_ARG(dtype == AB2_F64 || dtype == AB2_F32, "values must be fp64 or fp32");
    AB2_CHECK_ARG(K >= 1 && K <= AB2_COMMITTEE_MAX_MEMBERS, "members: 1 .. AB2_COMMITTEE_MAX_MEMBERS");
    AB2_CHECK_ARG(G >= 1 && m >= 0, "sizes");
    AB2_CHECK_ARG(x != nullptr, "null member table");
    if (m == 0) return 0;  // empty fields may come with null data pointers
    AB2_CHECK_ARG(mean != nullptr && dev != nullptr, "null pointer");
    CmMembers p;
    for (int k = 0; k < AB2_COMMITTEE_MAX_MEMBERS; ++k) p.p[k] = nullptr;
    for (int k = 0; k < K; ++k) {
        AB2_CHECK_ARG(x[k] != nullptr, "null member pointer");
        p.p[k] = x[k];
    }
    AB2_CHECK_ARG((m + CM_THREADS - 1) / CM_THREADS <= 0x7fffffffLL, "too many elements for one launch");
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == AB2_F64)
        committee_moments_kernel<double><<<ab2_blocks(m, CM_THREADS), CM_THREADS, 0, st>>>(K, m, G, p, (double*)mean, (double*)dev);
    else
        committee_moments_kernel<float><<<ab2_blocks(m, CM_THREADS), CM_THREADS, 0, st>>>(K, m, G, p, (float*)mean, (float*)dev);
    AB2_CUDA_LAUNCH_CHECK();
    return 0;
}

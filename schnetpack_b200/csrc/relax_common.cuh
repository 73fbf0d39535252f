// Device code shared by the batchwise optimizers: L-BFGS (relax.cu), FIRE (fire.cu) and the NEB forces that drive FIRE
// (neb.cu).  The fixed-order fp64 3-dot, the optimizer-unit force of an atom, and the convergence record and the
// unconverged count, which spk_lbfgs_t and spk_fire_t keep in fields of the same names.
#pragma once
#include "common.cuh"

namespace {

// x . y of two 3-vectors summed as numpy does along the last axis: (x0 y0 + x1 y1) + x2 y2, no contraction
__device__ __forceinline__ double dot3_rn(double x0, double x1, double x2, double y0, double y1, double y2) {
    return __dadd_rn(__dadd_rn(__dmul_rn(x0, y0), __dmul_rn(x1, y1)), __dmul_rn(x2, y2));
}

// force component c of atom a in optimizer units, zero on a fixed atom (get_forces, batchwise_optimization.py:196-197)
__device__ __forceinline__ double optimizer_force(bool fixed, const float* __restrict__ forces, double conversion,
                                                  int64_t a, int c) {
    return fixed ? 0.0 : (double)forces[3 * a + c] * conversion;
}

// the convergence record of system m from its largest squared force: fmax_sys, the converged flag and the step count at
// which the system became converged (kept while it stays converged, -1 while it is not).  max_sq is taken by reference
// so that the comparison compiles as it does written inline in a kernel (by value, the compiler swaps its operands).
template <class S>
__device__ __forceinline__ void record_convergence(const S& st, int64_t m, const double& max_sq) {
    const double fm = *st.fmax;
    const bool conv = max_sq < fm * fm;
    st.fmax_sys[m] = sqrt(max_sq);
    st.converged[m] = conv ? 1 : 0;
    const int64_t prev = st.steps[m];
    st.steps[m] = conv ? (prev >= 0 ? prev : st.counter[1]) : -1;
}

// count of unconverged systems (one CTA of 256 threads); the step counter read by the next step catches up with the one
// the last step wrote
template <class S>
__global__ void __launch_bounds__(256) k_count_unconverged(S st) {
    __shared__ int red[8];
    SPK_PDL_ENTER();
    int cnt = 0;
    for (int64_t m = threadIdx.x; m < st.n_sys; m += 256) cnt += st.converged[m] ? 0 : 1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int k = 0; k < 8; ++k) t += red[k];
        *st.n_unconverged = t;
        st.counter[0] = st.counter[1];
    }
}

}  // namespace

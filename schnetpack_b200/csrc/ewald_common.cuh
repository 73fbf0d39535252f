// Per-system cell records and fractional coordinates shared by the reciprocal terms of ewald.cu (Ewald sum) and pme.cu
// (smooth particle-mesh Ewald).
#pragma once
#include <math.h>

#include "common.cuh"
#include "segscan.cuh"

namespace {

constexpr int EW_SYS = 16;           // doubles per system record: H [9], V
constexpr double EW_PI = 3.14159265358979323846;

// H = h^-1 by cofactors and V = |det h| per system, fp64
__global__ void k_ewald_cell(const float* __restrict__ cell, int64_t n_sys, double* __restrict__ sys) {
    SPK_PDL_ENTER();
    const int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (m >= n_sys) return;
    double h[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) h[c] = cell[9 * m + c];
    const double c00 = h[4] * h[8] - h[5] * h[7], c01 = h[5] * h[6] - h[3] * h[8], c02 = h[3] * h[7] - h[4] * h[6];
    const double det = h[0] * c00 + h[1] * c01 + h[2] * c02;
    const double inv = 1.0 / det;
    double* o = sys + EW_SYS * m;
    o[0] = c00 * inv, o[1] = (h[2] * h[7] - h[1] * h[8]) * inv, o[2] = (h[1] * h[5] - h[2] * h[4]) * inv;
    o[3] = c01 * inv, o[4] = (h[0] * h[8] - h[2] * h[6]) * inv, o[5] = (h[2] * h[3] - h[0] * h[5]) * inv;
    o[6] = c02 * inv, o[7] = (h[1] * h[6] - h[0] * h[7]) * inv, o[8] = (h[0] * h[4] - h[1] * h[3]) * inv;
    o[9] = fabs(det);
}

// s_i = r_i H mod 1
__global__ void k_ewald_frac(const float* __restrict__ R, const int64_t* __restrict__ idx_m,
                             const double* __restrict__ sys, int64_t n_atoms, double* __restrict__ frac) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const double* H = sys + EW_SYS * idx_m[a];
    const double x = R[3 * a], y = R[3 * a + 1], z = R[3 * a + 2];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double s = x * H[c] + y * H[3 + c] + z * H[6 + c];
        frac[3 * a + c] = s - floor(s);
    }
}

// fixed tree over the SEG_FIN_T threads of a CTA; red[c][0] holds the totals on return
template <int NV>
__device__ __forceinline__ void ew_tree(double (&acc)[NV], double (*red)[SEG_FIN_T]) {
    const int t = threadIdx.x;
#pragma unroll
    for (int c = 0; c < NV; ++c) red[c][t] = acc[c];
    __syncthreads();
#pragma unroll
    for (int d = SEG_FIN_T / 2; d > 0; d >>= 1) {
        if (t < d) {
#pragma unroll
            for (int c = 0; c < NV; ++c) red[c][t] += red[c][t + d];
        }
        __syncthreads();
    }
}

}  // namespace

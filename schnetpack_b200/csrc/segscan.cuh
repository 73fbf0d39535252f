// Fixed-shape segmented reduction for deterministic per-system fp64 sums without atomics (used by the per-system virial in
// geometry.cu and the kinetic-energy sums of barostat.cu): CTAs of T consecutive items scan their items segment by segment
// and leave one partial per (system, CTA) pair; a per-system pass adds a system's partials in CTA order.
#pragma once
#include "common.cuh"

namespace {

// Inclusive segmented scan (Hillis-Steele) of NV fp64 values over the T threads of a CTA; f = 1 marks a segment head.
// The addition tree depends only on the segment layout, so the sums are bitwise reproducible.  sv / sf: shared scratch.
template <int T, int NV>
__device__ __forceinline__ void seg_scan(double (&v)[NV], int f, double (*sv)[T], int* sf) {
    const int t = threadIdx.x;
#pragma unroll
    for (int c = 0; c < NV; ++c) sv[c][t] = v[c];
    sf[t] = f;
    __syncthreads();
#pragma unroll
    for (int d = 1; d < T; d <<= 1) {
        double nv[NV];
        int nf = f;
#pragma unroll
        for (int c = 0; c < NV; ++c) nv[c] = v[c];
        if (t >= d) {
            if (!f) {
#pragma unroll
                for (int c = 0; c < NV; ++c) nv[c] = sv[c][t - d] + v[c];
            }
            nf = f | sf[t - d];
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < NV; ++c) sv[c][t] = v[c] = nv[c];
        sf[t] = f = nf;
        __syncthreads();
    }
}

// Per-system totals of NV-wide CTA partials, one CTA of SEG_FIN_T threads per system: the system's partials -- item 0 is
// the partial of the CTA in which it starts (sys_part[s]), item k >= 1 the head of the k-th later CTA it spans -- are
// summed by thread t over the items k = t, t + SEG_FIN_T, ... in ascending order, then by a fixed shared-memory tree.  The
// order depends only on the layout, so the totals are bitwise reproducible, and a system spanning a thousand CTAs costs a
// few strided loads per thread instead of a thousand dependent loads in one thread.  Items of system s are [i0, i1) with
// i(s) = ptr[outer[s]] (outer given) or ptr[s]; CTAs of the partial pass hold T items.  out[s * NV + c], 0 for no items.
constexpr int SEG_FIN_T = 128;

// The reduction of k_seg_finish for system s by the SEG_FIN_T threads of a CTA; red[c][0] holds the totals on return.
template <int T, int NV>
__device__ __forceinline__ void seg_finish_block(const int32_t* __restrict__ ptr, const int32_t* __restrict__ outer,
                                                 const double* __restrict__ sys_part, const double* __restrict__ head,
                                                 int64_t s, double (*red)[SEG_FIN_T]) {
    const int t = threadIdx.x;
    const int64_t i0 = outer ? ptr[outer[s]] : ptr[s];
    const int64_t i1 = outer ? ptr[outer[s + 1]] : ptr[s + 1];
    const int64_t n_items = i1 > i0 ? (i1 - 1) / T - i0 / T + 1 : 0;
    double acc[NV];
#pragma unroll
    for (int c = 0; c < NV; ++c) acc[c] = 0.0;
    for (int64_t k = t; k < n_items; k += SEG_FIN_T) {
        const double* src = k == 0 ? sys_part + s * NV : head + (i0 / T + k) * NV;
#pragma unroll
        for (int c = 0; c < NV; ++c) acc[c] += src[c];
    }
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

template <int T, int NV>
__global__ void __launch_bounds__(SEG_FIN_T) k_seg_finish(const int32_t* __restrict__ ptr, const int32_t* __restrict__ outer,
                                                          const double* __restrict__ sys_part,
                                                          const double* __restrict__ head, double* __restrict__ out) {
    __shared__ double red[NV][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x;
    seg_finish_block<T, NV>(ptr, outer, sys_part, head, s, red);
    if (threadIdx.x < NV) out[s * NV + threadIdx.x] = red[threadIdx.x][0];
}

}  // namespace

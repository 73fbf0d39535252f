// Fixed-shape segmented reduction for deterministic per-system fp64 sums without atomics, used by every per-system sum of
// the library: the kinetic energies of thermostat.cu, the kinetic-energy sums of barostat.cu, the centroid and barostat
// sums of rpmd.cu, the virial of geometry.cu and the dipole / polarizability assembly of equivariant.cu.  CTAs of T
// consecutive items scan their items segment by segment and leave one partial per (system, CTA) pair (seg_partials); a
// per-system pass adds a system's partials in CTA order (seg_finish_block, k_seg_finish).
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

// The same scan over the 32 lanes of warp 0 by shuffles: the addition tree of seg_scan for T <= 32 items, without shared
// memory or block barriers.
template <int NV>
__device__ __forceinline__ void seg_scan_warp(double (&v)[NV], int f) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int fu = __shfl_up_sync(0xffffffffu, f, d);
        double up[NV];
#pragma unroll
        for (int c = 0; c < NV; ++c) up[c] = __shfl_up_sync(0xffffffffu, v[c], d);
        if (lane >= d) {
            if (!f) {
#pragma unroll
                for (int c = 0; c < NV; ++c) v[c] += up[c];
            }
            f |= fu;
        }
    }
}

// The partial pass for the CTA of items [b0, b0 + T), b0 = blockIdx.x * T.  Thread t holds the NV terms v of item
// i = b0 + t (zeros if i >= n_items) and, for a valid item, its system m with items [first, end).  Each segment's total is
// the (system, CTA) partial: it goes to sys_part + m * NV if the system starts in this CTA, else to head + blockIdx.x * NV
// (only a CTA's first segment can continue a system).  Every thread of the CTA calls it (blockDim.x == T), or for T <= 32
// the 32 threads of warp 0 only.
template <int T, int NV>
__device__ __forceinline__ void seg_partials(double (&v)[NV], int64_t n_items, int64_t m, int64_t first, int64_t end,
                                             double* __restrict__ sys_part, double* __restrict__ head) {
    const int t = threadIdx.x;
    const int64_t b0 = (int64_t)blockIdx.x * T;
    const int64_t i = b0 + t;
    const bool item = t < T && i < n_items;
    const int f = !item || t == 0 || i == first;
    // the segment's last item writes its total; both are decided before the scan, so that m, first and end are not live
    // across it
    const bool last = item && (t == T - 1 || i == n_items - 1 || i + 1 == end);
    double* dst = first >= b0 ? sys_part + m * NV : head + (int64_t)blockIdx.x * NV;
    if constexpr (T <= 32) {
        seg_scan_warp<NV>(v, f);
    } else {
        __shared__ double sv[NV][T];
        __shared__ int sf[T];
        seg_scan<T, NV>(v, f, sv, sf);
    }
    if (!last) return;
#pragma unroll
    for (int c = 0; c < NV; ++c) dst[c] = v[c];
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

// Shared device helpers of the PaiNN edge kernels (painn.cu: LDG/LDS variant, painn_tma.cu: TMA + mbarrier pipeline).
#pragma once
#include "common.cuh"

// Filter weights of one channel as k-PAIRS (w[2m], w[2m+1]): with the radial basis read from shared memory as natural
// (phi[2m], phi[2m+1]) pairs, one spk_fma2 advances an even-k and an odd-k partial sum (two independent dependency chains);
// the two partials are added at the end.
template <int NRB>
struct FilterRegs {
    float2 a[NRB / 2], b[NRB / 2], c[NRB / 2];
    float ba, bb, bc;
};

template <int NRB>
__device__ __forceinline__ void load_filter(FilterRegs<NRB>& w, const float* __restrict__ wf,
                                            const float* __restrict__ bf, int F, int n_rbf, int c) {
#pragma unroll
    for (int m = 0; m < NRB / 2; ++m) {
        const int k0 = 2 * m, k1 = 2 * m + 1;
        const bool ok0 = k0 < n_rbf, ok1 = k1 < n_rbf;
        w.a[m] = make_float2(ok0 ? wf[(int64_t)c * n_rbf + k0] : 0.f, ok1 ? wf[(int64_t)c * n_rbf + k1] : 0.f);
        w.b[m] = make_float2(ok0 ? wf[(int64_t)(F + c) * n_rbf + k0] : 0.f, ok1 ? wf[(int64_t)(F + c) * n_rbf + k1] : 0.f);
        w.c[m] = make_float2(ok0 ? wf[(int64_t)(2 * F + c) * n_rbf + k0] : 0.f,
                             ok1 ? wf[(int64_t)(2 * F + c) * n_rbf + k1] : 0.f);
    }
    w.ba = bf[c];
    w.bb = bf[F + c];
    w.bc = bf[2 * F + c];
}


// Sum over the 32 lanes of 16 values per lane (4 edges x 4 scalars) with a transposing butterfly: 16 shuffles instead of
// 80.  Afterwards lane l holds the complete sum of value index 8*bit4 + 4*bit3 + 2*bit2 + bit1 (both lanes of a pair).
__device__ __forceinline__ float butterfly16(float (&v)[16], int lane) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const bool up = lane & 16;
        const float send = up ? v[i] : v[i + 8];
        const float keep = up ? v[i + 8] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const bool up = lane & 8;
        const float send = up ? v[i] : v[i + 4];
        const float keep = up ? v[i + 4] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const bool up = lane & 4;
        const float send = up ? v[i] : v[i + 2];
        const float keep = up ? v[i + 2] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    {
        const bool up = lane & 2;
        const float send = up ? v[0] : v[1];
        const float keep = up ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}

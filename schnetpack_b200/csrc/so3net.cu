// SO3net kernels (representation/so3net.py:136-146, nn/so3.py:177-334 of the reference): the fused SO3Convolution over
// the receiver CSR and its reverse grouped by sender, plus the per-atom self tensor product and gate with their reverses.
//
// Edge kernels: one CTA = ceil(F/32) warps, thread c owns feature channel c of every row s of a feature tensor
// [N, S, F] (S = (L+1)^2).  Its (L+1) x n_rbf filter weights stay in registers for the lifetime of the CTA, so the filter
// W[l, c] = fc (phi . wf[l F + c] + bf[l F + c]) is recomputed per edge and never stored.  The harmonics Y(u_e) (and
// dY/du in the reverse) of a chunk of edges are evaluated once per edge into shared memory; the sender row x[j] is
// gathered once per edge (S coalesced 4 F-byte rows) and the Clebsch-Gordan contraction runs from compile-time tables
// (so3_tables.cuh) into S register accumulators, in the table's fixed order.  A receiver's edges are reduced privately in
// CSR order (no atomics); CTAs take edge-balanced contiguous row ranges, as in painn.cu.
#include "common.cuh"
#include "so3_tables.cuh"

namespace {

constexpr int SO3_CH = 16;          // edges staged per chunk
constexpr int SO3_MAX_THREADS = 256;
constexpr int SO3_MAX_WARPS = SO3_MAX_THREADS / 32;

__host__ __device__ constexpr int so3_l(int s) {
    int l = 0;
    while ((l + 1) * (l + 1) <= s) ++l;
    return l;
}

// Y_s(u) = poly_s(z) T_m(x, y), T_m = Re (x+iy)^m (m > 0), Im (x+iy)^|m| (m < 0), 1 (m = 0); with GRAD also dY_s/du.
template <int L, bool GRAD>
__device__ __forceinline__ void so3_sh(float x, float y, float z, float* Y, float* dY) {
    float re[L + 1], im[L + 1];
    re[0] = 1.f;
    im[0] = 0.f;
#pragma unroll
    for (int m = 1; m <= L; ++m) {
        re[m] = x * re[m - 1] - y * im[m - 1];
        im[m] = x * im[m - 1] + y * re[m - 1];
    }
    So3Tab<L>::sh([&](int s, int m, float c0, float c1, float c2, float c3) {
        const int am = m < 0 ? -m : m;
        const int am1 = am > 0 ? am - 1 : 0;
        const float P = fmaf(fmaf(fmaf(c3, z, c2), z, c1), z, c0);
        const float T = m > 0 ? re[am] : (m < 0 ? im[am] : 1.f);
        Y[s] = P * T;
        if (GRAD) {
            const float dP = fmaf(fmaf(3.f * c3, z, 2.f * c2), z, c1);
            float Tx = 0.f, Ty = 0.f;
            if (m > 0) {
                Tx = am * re[am1];
                Ty = -am * im[am1];
            } else if (m < 0) {
                Tx = am * im[am1];
                Ty = am * re[am1];
            }
            dY[3 * s + 0] = P * Tx;
            dY[3 * s + 1] = P * Ty;
            dY[3 * s + 2] = dP * T;
        }
    });
}

// Filter weights of channel c: NRB > 0 -> registers (n_rbf <= NRB), NRB == 0 -> read through L1 (any n_rbf).
template <int L, int NRB>
struct So3Filter {
    float w[L + 1][NRB > 0 ? NRB : 1];
    float b[L + 1];
    const float* wf;
    int n_rbf, F, c;

    __device__ __forceinline__ void load(const float* __restrict__ wf_, const float* __restrict__ bf, int F_, int n_rbf_,
                                         int c_, bool active) {
        wf = wf_;
        n_rbf = n_rbf_;
        F = F_;
        c = active ? c_ : 0;
#pragma unroll
        for (int l = 0; l <= L; ++l) {
            b[l] = active ? bf[l * F + c] : 0.f;
            if (NRB > 0) {
#pragma unroll
                for (int k = 0; k < (NRB > 0 ? NRB : 1); ++k)
                    w[l][k] = (active && k < n_rbf) ? wf[(int64_t)(l * F + c) * n_rbf + k] : 0.f;
            }
        }
    }
    // P[l] = phi . w[l] + b[l]  (phi: NRB floats of shared memory, or n_rbf floats of global memory for NRB == 0)
    __device__ __forceinline__ void eval(const float* __restrict__ phi, float (&P)[L + 1]) const {
#pragma unroll
        for (int l = 0; l <= L; ++l) {
            float a0 = b[l], a1 = 0.f;
            if (NRB > 0) {
#pragma unroll
                for (int k = 0; k < (NRB > 0 ? NRB : 1); k += 2) {
                    a0 = fmaf(phi[k], w[l][k], a0);
                    a1 = fmaf(phi[k + 1], w[l][k + 1], a1);
                }
            } else {
                const float* __restrict__ wr = wf + (int64_t)(l * F + c) * n_rbf;
                for (int k = 0; k < n_rbf; ++k) a0 = fmaf(phi[k], __ldg(wr + k), a0);
            }
            P[l] = a0 + a1;
        }
    }
    // dP[l] = dphi . w[l]
    __device__ __forceinline__ void eval_nobias(const float* __restrict__ dphi, float (&P)[L + 1]) const {
#pragma unroll
        for (int l = 0; l <= L; ++l) {
            float a0 = 0.f, a1 = 0.f;
            if (NRB > 0) {
#pragma unroll
                for (int k = 0; k < (NRB > 0 ? NRB : 1); k += 2) {
                    a0 = fmaf(dphi[k], w[l][k], a0);
                    a1 = fmaf(dphi[k + 1], w[l][k + 1], a1);
                }
            } else {
                const float* __restrict__ wr = wf + (int64_t)(l * F + c) * n_rbf;
                for (int k = 0; k < n_rbf; ++k) a0 = fmaf(dphi[k], __ldg(wr + k), a0);
            }
            P[l] = a0 + a1;
        }
    }
};

// stage per-slot records [KP] of slot s into smem [NRB] (zero padded); NRB == 0 stages nothing
template <int NRB>
__device__ __forceinline__ void so3_stage_row(float* __restrict__ dst, const float* __restrict__ src, int KP, int q) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q * 4 < KP) v = *reinterpret_cast<const float4*>(src + q * 4);
    *reinterpret_cast<float4*>(dst + q * 4) = v;
}

template <int L, int NRB>
__global__ void __launch_bounds__(SO3_MAX_THREADS, 1) k_so3_conv_fwd(
    const float* __restrict__ x, const float* __restrict__ phi, const float* __restrict__ geo,
    const int* __restrict__ rowptr, const int* __restrict__ slot_j, const float* __restrict__ wf,
    const float* __restrict__ bf, int n_atoms, int n_edges, int F, int n_rbf, float* __restrict__ y) {
    SPK_PDL_ENTER();
    constexpr int S = (L + 1) * (L + 1);
    constexpr int NRS = NRB > 0 ? NRB : 4;
    __shared__ __align__(16) float s_phi[SO3_CH * NRS];
    __shared__ float s_Y[SO3_CH][S];
    __shared__ float s_fc[SO3_CH];
    __shared__ int s_j[SO3_CH];

    const int c = threadIdx.x;
    const bool active = c < F;
    const int nb = gridDim.x, b = blockIdx.x;
    const int row_lo = spk_block_row_begin(rowptr, n_atoms, n_edges, nb, b);
    const int row_hi = spk_block_row_begin(rowptr, n_atoms, n_edges, nb, b + 1);
    if (row_lo >= row_hi) return;

    So3Filter<L, NRB> w;
    w.load(wf, bf, F, n_rbf, c, active);
    const int KP = spk_kp(n_rbf);

    float acc[S];
#pragma unroll
    for (int s = 0; s < S; ++s) acc[s] = 0.f;
    auto flush = [&](int row) {
        if (active) {
#pragma unroll
            for (int s = 0; s < S; ++s) y[((int64_t)row * S + s) * F + c] = acc[s];
        }
#pragma unroll
        for (int s = 0; s < S; ++s) acc[s] = 0.f;
    };

    const int s_begin = rowptr[row_lo], s_end = rowptr[row_hi];
    int i = row_lo;
    int next_boundary = rowptr[i + 1];
    for (int cs = s_begin; cs < s_end; cs += SO3_CH) {
        const int n = min(SO3_CH, s_end - cs);
        __syncthreads();
        if (NRB > 0)
            for (int t = threadIdx.x; t < n * (NRS / 4); t += blockDim.x)
                so3_stage_row<NRB>(s_phi + (t / (NRS / 4)) * NRS, phi + (int64_t)(cs + t / (NRS / 4)) * KP, KP,
                                   t % (NRS / 4));
        if (threadIdx.x < n) {
            const int t = threadIdx.x;
            const float4 g = *reinterpret_cast<const float4*>(geo + (int64_t)(cs + t) * SPK_GEO_STRIDE);   // ux uy uz d
            float Yt[S];
            so3_sh<L, false>(g.x, g.y, g.z, Yt, nullptr);
#pragma unroll
            for (int s = 0; s < S; ++s) s_Y[t][s] = Yt[s];
            s_fc[t] = geo[(int64_t)(cs + t) * SPK_GEO_STRIDE + 4];
            s_j[t] = slot_j[cs + t];
        }
        __syncthreads();

        for (int t = 0; t < n; ++t) {
            const int sl = cs + t;
            while (sl >= next_boundary) {
                flush(i);
                ++i;
                next_boundary = rowptr[i + 1];
            }
            if (!active) continue;
            float xj[S];
            const float* __restrict__ xr = x + (int64_t)s_j[t] * S * F + c;
#pragma unroll
            for (int s = 0; s < S; ++s) xj[s] = xr[(int64_t)s * F];
            float P[L + 1];
            w.eval(NRB > 0 ? s_phi + t * NRS : phi + (int64_t)sl * KP, P);
            const float fc = s_fc[t];
            float wy[S];
#pragma unroll
            for (int s = 0; s < S; ++s) wy[s] = fc * P[so3_l(s)] * s_Y[t][s];
            So3Tab<L>::cg([&](int s1, int s2, int so, float C) { acc[so] = fmaf(C * wy[s1], xj[s2], acc[so]); });
        }
    }
    for (; i < row_hi; ++i) flush(i);
}

template <int L, int NRB>
__global__ void __launch_bounds__(SO3_MAX_THREADS, 1) k_so3_conv_bwd(
    const float* __restrict__ x, const float* __restrict__ g_y, const float* __restrict__ phi,
    const float* __restrict__ dphi, const float* __restrict__ geo, const int* __restrict__ sptr,
    const int* __restrict__ pos_slot, const int* __restrict__ pos_i, const int* __restrict__ slot_eid,
    const float* __restrict__ wf, const float* __restrict__ bf, int n_atoms, int n_edges, int F, int n_rbf,
    const float* __restrict__ g_res, float* __restrict__ g_x, float* __restrict__ g_rij, int accumulate) {
    SPK_PDL_ENTER();
    constexpr int S = (L + 1) * (L + 1);
    constexpr int NRS = NRB > 0 ? NRB : 4;
    __shared__ __align__(16) float s_phi[SO3_CH * NRS];
    __shared__ __align__(16) float s_dphi[SO3_CH * NRS];
    __shared__ float s_Y[SO3_CH][S];
    __shared__ float s_dY[SO3_CH][3 * S];
    __shared__ float s_geo[SO3_CH][8];
    __shared__ int s_i[SO3_CH];
    __shared__ int s_eid[SO3_CH];
    __shared__ int s_slot[SO3_CH];
    __shared__ float s_red[SO3_CH][SO3_MAX_WARPS][S + 1];

    const int c = threadIdx.x;
    const int lane = c & 31, warp = c >> 5, nw = blockDim.x >> 5;
    const bool active = c < F;
    const int nb = gridDim.x, b = blockIdx.x;
    const int j_lo = spk_block_row_begin(sptr, n_atoms, n_edges, nb, b);
    const int j_hi = spk_block_row_begin(sptr, n_atoms, n_edges, nb, b + 1);
    if (j_lo >= j_hi) return;

    So3Filter<L, NRB> w;
    w.load(wf, bf, F, n_rbf, c, active);
    const int KP = spk_kp(n_rbf);

    float xj[S], gx[S];
    auto load_own = [&](int row) {
#pragma unroll
        for (int s = 0; s < S; ++s) xj[s] = active ? x[((int64_t)row * S + s) * F + c] : 0.f;
    };
    auto flush = [&](int row) {
        if (active && g_x) {
#pragma unroll
            for (int s = 0; s < S; ++s) {
                const int64_t o = ((int64_t)row * S + s) * F + c;
                g_x[o] = (g_res ? g_res[o] : 0.f) + gx[s];
            }
        }
#pragma unroll
        for (int s = 0; s < S; ++s) gx[s] = 0.f;
    };
#pragma unroll
    for (int s = 0; s < S; ++s) gx[s] = 0.f;

    const int p_begin = sptr[j_lo], p_end = sptr[j_hi];
    int j = j_lo;
    int next_boundary = sptr[j + 1];
    load_own(j);
    for (int cs = p_begin; cs < p_end; cs += SO3_CH) {
        const int n = min(SO3_CH, p_end - cs);
        __syncthreads();
        if (threadIdx.x < n) s_slot[threadIdx.x] = pos_slot[cs + threadIdx.x];
        __syncthreads();
        if (NRB > 0)
            for (int t = threadIdx.x; t < n * (NRS / 4); t += blockDim.x) {
                const int r = t / (NRS / 4), q = t % (NRS / 4);
                so3_stage_row<NRB>(s_phi + r * NRS, phi + (int64_t)s_slot[r] * KP, KP, q);
                so3_stage_row<NRB>(s_dphi + r * NRS, dphi + (int64_t)s_slot[r] * KP, KP, q);
            }
        if (threadIdx.x < n) {
            const int t = threadIdx.x;
            const float* gr = geo + (int64_t)s_slot[t] * SPK_GEO_STRIDE;
#pragma unroll
            for (int k = 0; k < 8; ++k) s_geo[t][k] = gr[k];
            float Yt[S], dYt[3 * S];
            so3_sh<L, true>(gr[0], gr[1], gr[2], Yt, dYt);
#pragma unroll
            for (int s = 0; s < S; ++s) s_Y[t][s] = Yt[s];
#pragma unroll
            for (int s = 0; s < 3 * S; ++s) s_dY[t][s] = dYt[s];
            s_i[t] = pos_i[cs + t];
            s_eid[t] = slot_eid[s_slot[t]];
        }
        __syncthreads();

        for (int t = 0; t < n; ++t) {
            const int p = cs + t;
            if (p >= next_boundary) {
                do {
                    flush(j);
                    ++j;
                    next_boundary = sptr[j + 1];
                } while (p >= next_boundary);
                load_own(j);
            }
            float red[S + 1];
#pragma unroll
            for (int v = 0; v <= S; ++v) red[v] = 0.f;
            if (active) {
                float gy[S];
                const float* __restrict__ gr = g_y + (int64_t)s_i[t] * S * F + c;
#pragma unroll
                for (int s = 0; s < S; ++s) gy[s] = gr[(int64_t)s * F];
                float P[L + 1], dP[L + 1];
                w.eval(NRB > 0 ? s_phi + t * NRS : phi + (int64_t)s_slot[t] * KP, P);
                w.eval_nobias(NRB > 0 ? s_dphi + t * NRS : dphi + (int64_t)s_slot[t] * KP, dP);
                const float fc = s_geo[t][4], dfc = s_geo[t][5];
                float wy[S], G[S];
#pragma unroll
                for (int s = 0; s < S; ++s) {
                    wy[s] = fc * P[so3_l(s)] * s_Y[t][s];
                    G[s] = 0.f;
                }
                So3Tab<L>::cg([&](int s1, int s2, int so, float C) {
                    const float tg = C * gy[so];
                    gx[s2] = fmaf(tg, wy[s1], gx[s2]);
                    G[s1] = fmaf(tg, xj[s2], G[s1]);
                });
                float gd = 0.f;
#pragma unroll
                for (int s = 0; s < S; ++s) {
                    const int l = so3_l(s);
                    red[s] = fc * P[l] * G[s];                                        // dE/dY_s
                    gd = fmaf(G[s] * s_Y[t][s], fmaf(dfc, P[l], fc * dP[l]), gd);     // dE/dd through W
                }
                red[S] = gd;
            }
#pragma unroll
            for (int v = 0; v <= S; ++v) {
                const float tot = spk_warp_sum(red[v]);
                if (lane == 0) s_red[t][warp][v] = tot;
            }
        }
        __syncthreads();
        if (threadIdx.x < n) {
            const int t = threadIdx.x;
            float gY[S + 1];
#pragma unroll
            for (int v = 0; v <= S; ++v) {
                float a = 0.f;
                for (int wv = 0; wv < nw; ++wv) a += s_red[t][wv][v];
                gY[v] = a;
            }
            float gu0 = 0.f, gu1 = 0.f, gu2 = 0.f;
#pragma unroll
            for (int s = 0; s < S; ++s) {
                gu0 = fmaf(gY[s], s_dY[t][3 * s + 0], gu0);
                gu1 = fmaf(gY[s], s_dY[t][3 * s + 1], gu1);
                gu2 = fmaf(gY[s], s_dY[t][3 * s + 2], gu2);
            }
            const float ux = s_geo[t][0], uy = s_geo[t][1], uz = s_geo[t][2], inv = s_geo[t][6];
            const float gd = gY[S];
            const float dot = gu0 * ux + gu1 * uy + gu2 * uz;
            float r0 = gd * ux + (gu0 - dot * ux) * inv;
            float r1 = gd * uy + (gu1 - dot * uy) * inv;
            float r2 = gd * uz + (gu2 - dot * uz) * inv;
            float* out = g_rij + (int64_t)s_eid[t] * 3;
            if (accumulate) {
                r0 += out[0];
                r1 += out[1];
                r2 += out[2];
            }
            out[0] = r0;
            out[1] = r1;
            out[2] = r2;
        }
    }
    for (; j < j_hi; ++j) flush(j);
}

// ---- per-atom kernels: thread per (atom, channel) -----------------------------------------------------------------
template <int L>
__global__ void k_so3_tp_fwd(const float* __restrict__ dx, const float* __restrict__ ddx, int64_t n_atoms, int F,
                             float* __restrict__ out) {
    SPK_PDL_ENTER();
    constexpr int S = (L + 1) * (L + 1);
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    const int64_t a = t / F;
    const int c = (int)(t - a * F);
    const int64_t base = a * S * F + c;
    float u[S], v[S], o[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
        u[s] = dx[base + (int64_t)s * F];
        v[s] = ddx[base + (int64_t)s * F];
        o[s] = 0.f;
    }
    So3Tab<L>::cg([&](int s1, int s2, int so, float C) { o[so] = fmaf(C * u[s1], v[s2], o[so]); });
#pragma unroll
    for (int s = 0; s < S; ++s) out[base + (int64_t)s * F] = u[s] + o[s];
}

template <int L>
__global__ void k_so3_tp_bwd(const float* __restrict__ g, const float* __restrict__ dx, const float* __restrict__ ddx,
                             int64_t n_atoms, int F, float* __restrict__ g_dx, float* __restrict__ g_ddx) {
    SPK_PDL_ENTER();
    constexpr int S = (L + 1) * (L + 1);
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    const int64_t a = t / F;
    const int c = (int)(t - a * F);
    const int64_t base = a * S * F + c;
    float gg[S], u[S], v[S], gu[S], gv[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
        gg[s] = g[base + (int64_t)s * F];
        u[s] = dx[base + (int64_t)s * F];
        v[s] = ddx[base + (int64_t)s * F];
        gu[s] = 0.f;
        gv[s] = 0.f;
    }
    So3Tab<L>::cg([&](int s1, int s2, int so, float C) {
        const float tg = C * gg[so];
        gu[s1] = fmaf(tg, v[s2], gu[s1]);
        gv[s2] = fmaf(tg, u[s1], gv[s2]);
    });
#pragma unroll
    for (int s = 0; s < S; ++s) {
        g_dx[base + (int64_t)s * F] = gg[s] + gu[s];
        g_ddx[base + (int64_t)s * F] = gv[s];
    }
}

__device__ __forceinline__ float so3_sigmoid(float h) { return 1.0f / (1.0f + expf(-h)); }

template <int L>
__global__ void k_so3_gate_fwd(const float* __restrict__ x, const float* __restrict__ h, int64_t n_atoms, int F,
                               float* __restrict__ y) {
    SPK_PDL_ENTER();
    constexpr int S = (L + 1) * (L + 1);
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    const int64_t a = t / F;
    const int c = (int)(t - a * F);
    float sg[L + 1];
#pragma unroll
    for (int l = 0; l <= L; ++l) sg[l] = so3_sigmoid(h[(a * (L + 1) + l) * F + c]);
    const int64_t base = a * S * F + c;
#pragma unroll
    for (int s = 0; s < S; ++s) y[base + (int64_t)s * F] = x[base + (int64_t)s * F] * sg[so3_l(s)];
}

template <int L>
__global__ void k_so3_gate_bwd(const float* __restrict__ g_y, const float* __restrict__ x, const float* __restrict__ h,
                               int64_t n_atoms, int F, float* __restrict__ g_x, float* __restrict__ g_x0,
                               float* __restrict__ g_h) {
    SPK_PDL_ENTER();
    constexpr int S = (L + 1) * (L + 1);
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    const int64_t a = t / F;
    const int c = (int)(t - a * F);
    float sg[L + 1], gs[L + 1];
#pragma unroll
    for (int l = 0; l <= L; ++l) {
        sg[l] = so3_sigmoid(h[(a * (L + 1) + l) * F + c]);
        gs[l] = 0.f;
    }
    const int64_t base = a * S * F + c;
#pragma unroll
    for (int s = 0; s < S; ++s) {
        const int l = so3_l(s);
        const float gy = g_y[base + (int64_t)s * F];
        gs[l] = fmaf(gy, x[base + (int64_t)s * F], gs[l]);
        if (s == 0)
            g_x0[a * F + c] = gy * sg[0];
        else
            g_x[base + (int64_t)s * F] = gy * sg[l];
    }
#pragma unroll
    for (int l = 0; l <= L; ++l) g_h[(a * (L + 1) + l) * F + c] = gs[l] * sg[l] * (1.f - sg[l]);
}

__global__ void k_so3_put_l0(const float* __restrict__ src, const float* __restrict__ v, int64_t n_atoms, int S, int F,
                             float* __restrict__ out) {
    SPK_PDL_ENTER();
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * S * F) return;
    const int64_t a = t / ((int64_t)S * F);
    const int64_t r = t - a * S * F;
    float o = src ? src[t] : 0.f;
    if (r < F && v) o += v[a * F + r];
    out[t] = o;
}

__global__ void k_so3_take_l0(const float* __restrict__ x, int64_t n_atoms, int S, int F, float* __restrict__ q) {
    SPK_PDL_ENTER();
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    const int64_t a = t / F;
    q[t] = x[a * S * F + (t - a * F)];
}

// one resident wave of CTAs (no tail), >= 32 edges per CTA, at most one CTA per atom
template <typename K>
int64_t so3_grid(K kernel, int threads, int64_t n_atoms, int64_t n_edges) {
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, 0);
    int64_t nb = (int64_t)spk_num_sms() * (occ < 1 ? 1 : occ);
    if (nb > spk_cdiv(n_edges, 32)) nb = spk_cdiv(n_edges, 32);
    if (nb < 1) nb = 1;
    if (nb > n_atoms) nb = n_atoms;
    return nb;
}

template <int L, int NRB>
void launch_conv_fwd(const float* x, const float* phi, const float* geo, const int32_t* rowptr, const int32_t* slot_j,
                     const float* wf, const float* bf, int64_t n_atoms, int64_t n_edges, int F, int n_rbf, float* y,
                     cudaStream_t st) {
    const int threads = (F + 31) & ~31;
    const int64_t nb = so3_grid(k_so3_conv_fwd<L, NRB>, threads, n_atoms, n_edges);
    spk_launch(k_so3_conv_fwd<L, NRB>, (unsigned)nb, threads, 0, st, x, phi, geo, rowptr, slot_j, wf, bf, (int)n_atoms,
               (int)n_edges, F, n_rbf, y);
}

template <int L, int NRB>
void launch_conv_bwd(const float* x, const float* g_y, const float* phi, const float* dphi, const float* geo,
                     const int32_t* sptr, const int32_t* pos_slot, const int32_t* pos_i, const int32_t* slot_eid,
                     const float* wf, const float* bf, int64_t n_atoms, int64_t n_edges, int F, int n_rbf,
                     const float* g_res, float* g_x, float* g_rij, int accumulate, cudaStream_t st) {
    const int threads = (F + 31) & ~31;
    const int64_t nb = so3_grid(k_so3_conv_bwd<L, NRB>, threads, n_atoms, n_edges);
    spk_launch(k_so3_conv_bwd<L, NRB>, (unsigned)nb, threads, 0, st, x, g_y, phi, dphi, geo, sptr, pos_slot, pos_i,
               slot_eid, wf, bf, (int)n_atoms, (int)n_edges, F, n_rbf, g_res, g_x, g_rij, accumulate);
}

bool so3_shape_ok(int lmax, int F) { return lmax >= 0 && lmax <= 3 && F > 0 && F % 4 == 0 && F <= SO3_MAX_THREADS; }

}  // namespace

#define SO3_DISPATCH_L(CALL)                   \
    do {                                       \
        switch (lmax) {                        \
            case 0: CALL(0); break;            \
            case 1: CALL(1); break;            \
            case 2: CALL(2); break;            \
            default: CALL(3); break;           \
        }                                      \
    } while (0)

// filter weights in registers for n_rbf <= 20 (<= 32 below lmax 3, where 32 would spill); otherwise read through L1
#define SO3_DISPATCH_L2(CALL)                  \
    do {                                       \
        switch (lmax) {                        \
            case 0: CALL(0); break;            \
            case 1: CALL(1); break;            \
            default: CALL(2); break;           \
        }                                      \
    } while (0)

#define SO3_DISPATCH_L_NRB(CALL)                                  \
    do {                                                          \
        if (n_rbf <= 20) { SO3_DISPATCH_L(CALL##_20); }           \
        else if (n_rbf <= 32 && lmax < 3) { SO3_DISPATCH_L2(CALL##_32); } \
        else { SO3_DISPATCH_L(CALL##_0); }                        \
    } while (0)

extern "C" int spk_so3_conv_fwd(const float* x, const float* phi, const float* geo, const int32_t* rowptr,
                                const int32_t* slot_j, const float* wf, const float* bf, int64_t n_atoms,
                                int64_t n_edges, int lmax, int F, int n_rbf, float* y, spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !rowptr || !wf || !bf || !y) return SPK_ERR_ARG;
    if (n_edges > 0 && (!phi || !geo || !slot_j)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
#define FWD_20(L) launch_conv_fwd<L, 20>(x, phi, geo, rowptr, slot_j, wf, bf, n_atoms, n_edges, F, n_rbf, y, st)
#define FWD_32(L) launch_conv_fwd<L, 32>(x, phi, geo, rowptr, slot_j, wf, bf, n_atoms, n_edges, F, n_rbf, y, st)
#define FWD_0(L) launch_conv_fwd<L, 0>(x, phi, geo, rowptr, slot_j, wf, bf, n_atoms, n_edges, F, n_rbf, y, st)
    SO3_DISPATCH_L_NRB(FWD);
#undef FWD_20
#undef FWD_32
#undef FWD_0
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_so3_conv_bwd(const float* x, const float* g_y, const float* phi, const float* dphi, const float* geo,
                                const int32_t* sptr, const int32_t* pos_slot, const int32_t* pos_i,
                                const int32_t* slot_eid, const float* wf, const float* bf, int64_t n_atoms,
                                int64_t n_edges, int lmax, int F, int n_rbf, const float* g_res, float* g_x,
                                float* g_rij, int accumulate, spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !g_y || !sptr || !wf || !bf) return SPK_ERR_ARG;
    if (n_edges > 0 && (!phi || !dphi || !geo || !pos_slot || !pos_i || !slot_eid || !g_rij)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
#define BWD_ARGS x, g_y, phi, dphi, geo, sptr, pos_slot, pos_i, slot_eid, wf, bf, n_atoms, n_edges, F, n_rbf, g_res, g_x, \
                 g_rij, accumulate, st
#define BWD_20(L) launch_conv_bwd<L, 20>(BWD_ARGS)
#define BWD_32(L) launch_conv_bwd<L, 32>(BWD_ARGS)
#define BWD_0(L) launch_conv_bwd<L, 0>(BWD_ARGS)
    SO3_DISPATCH_L_NRB(BWD);
#undef BWD_20
#undef BWD_32
#undef BWD_0
#undef BWD_ARGS
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

#define SO3_GRID(n) (unsigned)spk_cdiv((n), 256), 256, 0, spk_st(stream)

extern "C" int spk_so3_tp_fwd(const float* dx, const float* ddx, int64_t n_atoms, int lmax, int F, float* out,
                              spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!dx || !ddx || !out) return SPK_ERR_ARG;
#define TPF(L) spk_launch(k_so3_tp_fwd<L>, SO3_GRID(n_atoms * F), dx, ddx, n_atoms, F, out)
    SO3_DISPATCH_L(TPF);
#undef TPF
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_so3_tp_bwd(const float* g, const float* dx, const float* ddx, int64_t n_atoms, int lmax, int F,
                              float* g_dx, float* g_ddx, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!g || !dx || !ddx || !g_dx || !g_ddx) return SPK_ERR_ARG;
#define TPB(L) spk_launch(k_so3_tp_bwd<L>, SO3_GRID(n_atoms * F), g, dx, ddx, n_atoms, F, g_dx, g_ddx)
    SO3_DISPATCH_L(TPB);
#undef TPB
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_so3_gate_fwd(const float* x, const float* h, int64_t n_atoms, int lmax, int F, float* y,
                                spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !h || !y) return SPK_ERR_ARG;
#define GF(L) spk_launch(k_so3_gate_fwd<L>, SO3_GRID(n_atoms * F), x, h, n_atoms, F, y)
    SO3_DISPATCH_L(GF);
#undef GF
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_so3_gate_bwd(const float* g_y, const float* x, const float* h, int64_t n_atoms, int lmax, int F,
                                float* g_x, float* g_x0, float* g_h, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!g_y || !x || !h || !g_x || !g_x0 || !g_h) return SPK_ERR_ARG;
#define GB(L) spk_launch(k_so3_gate_bwd<L>, SO3_GRID(n_atoms * F), g_y, x, h, n_atoms, F, g_x, g_x0, g_h)
    SO3_DISPATCH_L(GB);
#undef GB
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_so3_put_l0(const float* src, const float* v, int64_t n_atoms, int lmax, int F, float* out,
                              spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!out) return SPK_ERR_ARG;
    const int S = (lmax + 1) * (lmax + 1);
    spk_launch(k_so3_put_l0, SO3_GRID(n_atoms * S * F), src, v, n_atoms, S, F, out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_so3_take_l0(const float* x, int64_t n_atoms, int lmax, int F, float* q, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (!so3_shape_ok(lmax, F)) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !q) return SPK_ERR_ARG;
    const int S = (lmax + 1) * (lmax + 1);
    spk_launch(k_so3_take_l0, SO3_GRID(n_atoms * F), x, n_atoms, S, F, q);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

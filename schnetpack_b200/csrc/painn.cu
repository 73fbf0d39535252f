// PaiNN interaction-block kernels: the fused per-edge pipeline (filter recomputed on the fly -> continuous-filter
// product -> equivariant scalar/vector mix -> segmented reduction to receivers) and its reverse (grouped by sender),
// plus the elementwise glue of PaiNNMixing.   Reference: representation/painn.py:31-67, :92-117, :227-236.
//
// Thread mapping: one "group" of F threads (F/32 warps) per CTA; thread c owns feature channel c of all three filter
// thirds (c, F+c, 2F+c).  Its 3*(n_rbf+1) filter weights live in registers for the lifetime of the CTA, the per-edge
// radial basis / geometry records of a chunk of edges are staged in shared memory (coalesced 128-bit loads) and read
// back as warp-broadcast LDS.128, sender rows x[j], mu[j] are gathered with fully coalesced 128 B requests, and the
// reduction over a receiver's edges is a private register accumulation (CSR order) -- no atomics, no shuffles.
// CTAs take edge-balanced contiguous row ranges (binary search in rowptr).
#include "painn_common.cuh"

namespace {

#ifndef SPK_EDGE_MINB
#define SPK_EDGE_MINB(NW) (512 / ((NW) * 32))   // resident CTAs per SM the register allocation is sized for
#endif
constexpr int CH = 32;   // edges staged per chunk (multiple of the 4-edge reduction groups of the reverse kernel)

// cooperative staging of contiguous per-slot records [n, KP] -> smem [n, NRB] (zero padded)
template <int NRB, int NTHR>
__device__ __forceinline__ void stage_rows_contig(float* __restrict__ dst, const float* __restrict__ src, int n, int KP) {
    const int kq = KP >> 2;
    for (int t = threadIdx.x; t < n * (NRB / 4); t += NTHR) {
        int r = t / (NRB / 4), q = t - r * (NRB / 4);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q < kq) v = *reinterpret_cast<const float4*>(src + (int64_t)r * KP + q * 4);
        *reinterpret_cast<float4*>(dst + r * NRB + q * 4) = v;
    }
}

template <int NW, int NRB, bool HAS_MU>
__global__ void __launch_bounds__(NW * 32, SPK_EDGE_MINB(NW)) k_painn_edge_fwd(
    const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ q,
    const float* __restrict__ phi, const float* __restrict__ geo, const int* __restrict__ rowptr,
    const int* __restrict__ slot_j, const float* __restrict__ wf, const float* __restrict__ bf, int n_atoms,
    int n_edges, int n_rbf, float* __restrict__ q_out, float* __restrict__ mu_out) {
    SPK_PDL_ENTER();
    constexpr int F = NW * 32;
    constexpr int NTHR = NW * 32;
    __shared__ __align__(16) float s_phi[CH * NRB];
    __shared__ __align__(16) float s_geo[CH * SPK_GEO_STRIDE];
    __shared__ int s_j[CH];

    const int c = threadIdx.x;
    const int nb = gridDim.x, b = blockIdx.x;
    const int row_lo = spk_block_row_begin(rowptr, n_atoms, n_edges, nb, b);
    const int row_hi = spk_block_row_begin(rowptr, n_atoms, n_edges, nb, b + 1);
    if (row_lo >= row_hi) return;

    FilterRegs<NRB> w;
    load_filter<NRB>(w, wf, bf, F, n_rbf, c);
    const int KP = spk_kp(n_rbf);

    const int s_begin = rowptr[row_lo], s_end = rowptr[row_hi];
    int i = row_lo;
    int next_boundary = rowptr[i + 1];
    float dq = 0.f, dm0 = 0.f, dm1 = 0.f, dm2 = 0.f;

    auto flush = [&](int row) {
        const size_t o = (size_t)row * F + c;
        q_out[o] = q[o] + dq;
        const size_t om = (size_t)row * 3 * F + c;
        if (HAS_MU) {
            mu_out[om] = mu[om] + dm0;
            mu_out[om + F] = mu[om + F] + dm1;
            mu_out[om + 2 * F] = mu[om + 2 * F] + dm2;
        } else {
            mu_out[om] = dm0;
            mu_out[om + F] = dm1;
            mu_out[om + 2 * F] = dm2;
        }
        dq = dm0 = dm1 = dm2 = 0.f;
    };

    for (int cs = s_begin; cs < s_end; cs += CH) {
        const int n = min(CH, s_end - cs);
        __syncthreads();
        stage_rows_contig<NRB, NTHR>(s_phi, phi + (int64_t)cs * KP, n, KP);
        for (int t = threadIdx.x; t < n * 2; t += NTHR)
            reinterpret_cast<float4*>(s_geo)[t] = reinterpret_cast<const float4*>(geo + (int64_t)cs * SPK_GEO_STRIDE)[t];
        for (int t = threadIdx.x; t < n; t += NTHR) s_j[t] = slot_j[cs + t];
        __syncthreads();

#pragma unroll 2
        for (int t = 0; t < n; ++t) {
            const int s = cs + t;
            while (s >= next_boundary) {
                flush(i);
                ++i;
                next_boundary = rowptr[i + 1];
            }
            float xa, xb, xc = 0.f, m0 = 0.f, m1 = 0.f, m2 = 0.f;
            {
                const int j = s_j[t];
                const float* __restrict__ xj = x + (size_t)j * (3 * F) + c;
                xa = xj[0];
                xb = xj[F];
                if (HAS_MU) {
                    xc = xj[2 * F];
                    const float* __restrict__ mj = mu + (size_t)j * (3 * F) + c;
                    m0 = mj[0];
                    m1 = mj[F];
                    m2 = mj[2 * F];
                }
            }
            const float4 g0 = *reinterpret_cast<const float4*>(s_geo + t * SPK_GEO_STRIDE);      // ux uy uz d
            const float fc = s_geo[t * SPK_GEO_STRIDE + 4];
            float2 pa2 = make_float2(w.ba, 0.f), pb2 = make_float2(w.bb, 0.f), pc2 = make_float2(w.bc, 0.f);
            const float4* __restrict__ ph = reinterpret_cast<const float4*>(s_phi + t * NRB);
#pragma unroll
            for (int k4 = 0; k4 < NRB / 4; ++k4) {
                const float4 p = ph[k4];
                const float2 p01 = make_float2(p.x, p.y), p23 = make_float2(p.z, p.w);
                pa2 = spk_fma2(p01, w.a[2 * k4], pa2);
                pb2 = spk_fma2(p01, w.b[2 * k4], pb2);
                pa2 = spk_fma2(p23, w.a[2 * k4 + 1], pa2);
                pb2 = spk_fma2(p23, w.b[2 * k4 + 1], pb2);
                if (HAS_MU) {
                    pc2 = spk_fma2(p01, w.c[2 * k4], pc2);
                    pc2 = spk_fma2(p23, w.c[2 * k4 + 1], pc2);
                }
            }
            const float pa = pa2.x + pa2.y, pb = pb2.x + pb2.y, pc = pc2.x + pc2.y;
            dq = fmaf(fc * pa, xa, dq);
            const float tb = fc * pb * xb;
            dm0 = fmaf(tb, g0.x, dm0);
            dm1 = fmaf(tb, g0.y, dm1);
            dm2 = fmaf(tb, g0.z, dm2);
            if (HAS_MU) {
                const float tc = fc * pc * xc;
                dm0 = fmaf(tc, m0, dm0);
                dm1 = fmaf(tc, m1, dm1);
                dm2 = fmaf(tc, m2, dm2);
            }
        }
    }
    for (; i < row_hi; ++i) flush(i);
}

// ------------------------------------------------------------------------------------------------------------------
// reverse pass, grouped by sender
// ------------------------------------------------------------------------------------------------------------------

template <int NW, int NRB, bool HAS_MU>
__global__ void __launch_bounds__(NW * 32, SPK_EDGE_MINB(NW)) k_painn_edge_bwd(
    const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ g_q,
    const float* __restrict__ g_mu, const float* __restrict__ phi, const float* __restrict__ dphi,
    const float* __restrict__ geo, const int* __restrict__ sptr, const int* __restrict__ pos_slot,
    const int* __restrict__ pos_i, const int* __restrict__ slot_eid, const float* __restrict__ wf,
    const float* __restrict__ bf, int n_atoms, int n_edges, int n_rbf, float* __restrict__ g_x,
    float* __restrict__ g_mu_in, float* __restrict__ g_rij, int accumulate) {
    SPK_PDL_ENTER();
    constexpr int F = NW * 32;
    constexpr int NTHR = NW * 32;
    __shared__ __align__(16) float s_phi[CH * NRB];
    __shared__ __align__(16) float s_dphi[CH * NRB];
    __shared__ __align__(16) float s_geo[CH * SPK_GEO_STRIDE];
    __shared__ int s_i[CH];
    __shared__ int s_eid[CH];
    __shared__ float s_red[CH][NW][4];

    const int c = threadIdx.x;
    const int lane = c & 31, warp = c >> 5;
    const int nb = gridDim.x, b = blockIdx.x;
    const int j_lo = spk_block_row_begin(sptr, n_atoms, n_edges, nb, b);
    const int j_hi = spk_block_row_begin(sptr, n_atoms, n_edges, nb, b + 1);
    if (j_lo >= j_hi) return;

    FilterRegs<NRB> w;
    load_filter<NRB>(w, wf, bf, F, n_rbf, c);
    const int KP = spk_kp(n_rbf);
    const int kq = KP >> 2;

    const int p_begin = sptr[j_lo], p_end = sptr[j_hi];
    int j = j_lo;
    int next_boundary = sptr[j + 1];
    float xa, xb, xc = 0.f, m0 = 0.f, m1 = 0.f, m2 = 0.f;
    float gxa = 0.f, gxb = 0.f, gxc = 0.f, gm0 = 0.f, gm1 = 0.f, gm2 = 0.f;

    auto load_own = [&](int row) {
        const float* __restrict__ xr = x + (size_t)row * (3 * F) + c;
        xa = xr[0];
        xb = xr[F];
        if (HAS_MU) {
            xc = xr[2 * F];
            const float* __restrict__ mr = mu + (size_t)row * (3 * F) + c;
            m0 = mr[0];
            m1 = mr[F];
            m2 = mr[2 * F];
        }
    };
    auto flush = [&](int row) {
        const size_t o = (size_t)row * 3 * F + c;
        g_x[o] = gxa;
        g_x[o + F] = gxb;
        g_x[o + 2 * F] = gxc;
        if (HAS_MU) {
            g_mu_in[o] = g_mu[o] + gm0;
            g_mu_in[o + F] = g_mu[o + F] + gm1;
            g_mu_in[o + 2 * F] = g_mu[o + 2 * F] + gm2;
        }
        gxa = gxb = gxc = gm0 = gm1 = gm2 = 0.f;
    };
    load_own(j);
    // value index held by this lane after the butterfly: edge (idx >> 2) of the group, scalar (idx & 3)
    const int my_idx = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);

    for (int cs = p_begin; cs < p_end; cs += CH) {
        const int n = min(CH, p_end - cs);
        __syncthreads();
        // gather the per-slot records of this chunk (random 16 B-aligned rows)
        for (int t = threadIdx.x; t < n * (NRB / 4); t += NTHR) {
            int r = t / (NRB / 4), qd = t - r * (NRB / 4);
            int s = pos_slot[cs + r];
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f), dv = v;
            if (qd < kq) {
                v = *reinterpret_cast<const float4*>(phi + (int64_t)s * KP + qd * 4);
                dv = *reinterpret_cast<const float4*>(dphi + (int64_t)s * KP + qd * 4);
            }
            *reinterpret_cast<float4*>(s_phi + r * NRB + qd * 4) = v;
            *reinterpret_cast<float4*>(s_dphi + r * NRB + qd * 4) = dv;
        }
        for (int t = threadIdx.x; t < n * 2; t += NTHR) {
            int r = t >> 1;
            int s = pos_slot[cs + r];
            reinterpret_cast<float4*>(s_geo)[t] = reinterpret_cast<const float4*>(geo + (int64_t)s * SPK_GEO_STRIDE)[t & 1];
        }
        for (int t = threadIdx.x; t < n; t += NTHR) {
            s_i[t] = pos_i[cs + t];
            s_eid[t] = slot_eid[pos_slot[cs + t]];
        }
        __syncthreads();

        for (int t0 = 0; t0 < n; t0 += 4) {
            float red[16];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int t = t0 + u;
                float part_d = 0.f, pu0 = 0.f, pu1 = 0.f, pu2 = 0.f;
                if (t < n) {
                    const int p = cs + t;
                    if (p >= next_boundary) {
                        do {
                            flush(j);
                            ++j;
                            next_boundary = sptr[j + 1];
                        } while (p >= next_boundary);
                        load_own(j);
                    }
                    float gq, g0, g1, g2;
                    {
                        const int i = s_i[t];
                        gq = g_q[(size_t)i * F + c];
                        const float* __restrict__ gmi = g_mu + (size_t)i * (3 * F) + c;
                        g0 = gmi[0];
                        g1 = gmi[F];
                        g2 = gmi[2 * F];
                    }
                    const float4 ge = *reinterpret_cast<const float4*>(s_geo + t * SPK_GEO_STRIDE);   // ux uy uz d
                    const float fc = s_geo[t * SPK_GEO_STRIDE + 4], dfc = s_geo[t * SPK_GEO_STRIDE + 5];
                    float2 pa2 = make_float2(w.ba, 0.f), pb2 = make_float2(w.bb, 0.f), pc2 = make_float2(w.bc, 0.f);
                    float2 da2 = make_float2(0.f, 0.f), db2 = da2, dc2 = da2;
                    const float4* __restrict__ ph = reinterpret_cast<const float4*>(s_phi + t * NRB);
                    const float4* __restrict__ dh = reinterpret_cast<const float4*>(s_dphi + t * NRB);
#pragma unroll
                    for (int k4 = 0; k4 < NRB / 4; ++k4) {
                        const float4 p4 = ph[k4];
                        const float4 d4 = dh[k4];
                        const float2 p01 = make_float2(p4.x, p4.y), p23 = make_float2(p4.z, p4.w);
                        const float2 d01 = make_float2(d4.x, d4.y), d23 = make_float2(d4.z, d4.w);
                        pa2 = spk_fma2(p01, w.a[2 * k4], pa2);
                        da2 = spk_fma2(d01, w.a[2 * k4], da2);
                        pb2 = spk_fma2(p01, w.b[2 * k4], pb2);
                        db2 = spk_fma2(d01, w.b[2 * k4], db2);
                        pa2 = spk_fma2(p23, w.a[2 * k4 + 1], pa2);
                        da2 = spk_fma2(d23, w.a[2 * k4 + 1], da2);
                        pb2 = spk_fma2(p23, w.b[2 * k4 + 1], pb2);
                        db2 = spk_fma2(d23, w.b[2 * k4 + 1], db2);
                        if (HAS_MU) {
                            pc2 = spk_fma2(p01, w.c[2 * k4], pc2);
                            dc2 = spk_fma2(d01, w.c[2 * k4], dc2);
                            pc2 = spk_fma2(p23, w.c[2 * k4 + 1], pc2);
                            dc2 = spk_fma2(d23, w.c[2 * k4 + 1], dc2);
                        }
                    }
                    const float pa = pa2.x + pa2.y, pb = pb2.x + pb2.y, pc = pc2.x + pc2.y;
                    const float da = da2.x + da2.y, db = db2.x + db2.y, dc = dc2.x + dc2.y;
                    const float Wa = fc * pa, Wb = fc * pb;
                    const float dWa = fmaf(dfc, pa, fc * da), dWb = fmaf(dfc, pb, fc * db);
                    const float gu = g0 * ge.x + g1 * ge.y + g2 * ge.z;   // sum_d g_mu[i,d] u_d
                    gxa = fmaf(Wa, gq, gxa);
                    gxb = fmaf(Wb, gu, gxb);
                    part_d = gq * xa * dWa + gu * xb * dWb;
                    const float wbx = Wb * xb;
                    pu0 = g0 * wbx;
                    pu1 = g1 * wbx;
                    pu2 = g2 * wbx;
                    if (HAS_MU) {
                        const float Wc = fc * pc;
                        const float dWc = fmaf(dfc, pc, fc * dc);
                        const float gm = g0 * m0 + g1 * m1 + g2 * m2;     // sum_d g_mu[i,d] mu[j,d]
                        gxc = fmaf(Wc, gm, gxc);
                        const float wcx = Wc * xc;
                        gm0 = fmaf(wcx, g0, gm0);
                        gm1 = fmaf(wcx, g1, gm1);
                        gm2 = fmaf(wcx, g2, gm2);
                        part_d = fmaf(gm * xc, dWc, part_d);
                    }
                }
                red[4 * u + 0] = part_d;
                red[4 * u + 1] = pu0;
                red[4 * u + 2] = pu1;
                red[4 * u + 3] = pu2;
            }
            const float tot = butterfly16(red, lane);
            const int te = t0 + (my_idx >> 2);
            if (!(lane & 1) && te < n) s_red[te][warp][my_idx & 3] = tot;
        }
        __syncthreads();
        if (threadIdx.x < n) {
            const int t = threadIdx.x;
            float gd = 0.f, u0 = 0.f, u1 = 0.f, u2 = 0.f;
#pragma unroll
            for (int wv = 0; wv < NW; ++wv) {
                gd += s_red[t][wv][0];
                u0 += s_red[t][wv][1];
                u1 += s_red[t][wv][2];
                u2 += s_red[t][wv][3];
            }
            const float ux = s_geo[t * SPK_GEO_STRIDE + 0], uy = s_geo[t * SPK_GEO_STRIDE + 1],
                        uz = s_geo[t * SPK_GEO_STRIDE + 2], inv = s_geo[t * SPK_GEO_STRIDE + 6];
            const float dot = u0 * ux + u1 * uy + u2 * uz;
            float r0 = gd * ux + (u0 - dot * ux) * inv;
            float r1 = gd * uy + (u1 - dot * uy) * inv;
            float r2 = gd * uz + (u2 - dot * uz) * inv;
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

// ------------------------------------------------------------------------------------------------------------------
// PaiNNMixing glue (painn.py:103-116); thread per (atom, channel); VW = mu_channel_mix(mu) [N,3,2F]
// ------------------------------------------------------------------------------------------------------------------
__global__ void k_mix_ctx(const float* __restrict__ q, const float* __restrict__ VW, int64_t n_atoms, int F, float eps,
                          float* __restrict__ ctx) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    int64_t a = t / F;
    int c = (int)(t - a * F);
    const float* v = VW + a * 6 * F + c;
    float v0 = v[0], v1 = v[2 * F], v2 = v[4 * F];
    ctx[a * 2 * F + c] = q[t];
    ctx[a * 2 * F + F + c] = sqrtf(v0 * v0 + v1 * v1 + v2 * v2 + eps);
}

__global__ void k_mix_update(const float* __restrict__ q, const float* __restrict__ mu, const float* __restrict__ s,
                             const float* __restrict__ VW, int64_t n_atoms, int F, float* __restrict__ q_out,
                             float* __restrict__ mu_out) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    int64_t a = t / F;
    int c = (int)(t - a * F);
    const float* vw = VW + a * 6 * F + c;
    float v0 = vw[0], w0 = vw[F], v1 = vw[2 * F], w1 = vw[3 * F], v2 = vw[4 * F], w2 = vw[5 * F];
    const float* sr = s + a * 3 * F + c;
    float s1 = sr[0], s2 = sr[F], s3 = sr[2 * F];
    float svw = v0 * w0 + v1 * w1 + v2 * w2;
    q_out[t] = q[t] + s1 + s3 * svw;
    int64_t om = a * 3 * F + c;
    mu_out[om] = mu[om] + s2 * w0;
    mu_out[om + F] = mu[om + F] + s2 * w1;
    mu_out[om + 2 * F] = mu[om + 2 * F] + s2 * w2;
}

__global__ void k_mix_update_bwd(const float* __restrict__ g_q, const float* __restrict__ g_mu,
                                 const float* __restrict__ s, const float* __restrict__ VW, int64_t n_atoms, int F,
                                 float* __restrict__ g_s, float* __restrict__ g_VW) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    int64_t a = t / F;
    int c = (int)(t - a * F);
    const float* vw = VW + a * 6 * F + c;
    float v0 = vw[0], w0 = vw[F], v1 = vw[2 * F], w1 = vw[3 * F], v2 = vw[4 * F], w2 = vw[5 * F];
    const float* sr = s + a * 3 * F + c;
    float s2 = sr[F], s3 = sr[2 * F];
    float gq = g_q[t];
    int64_t om = a * 3 * F + c;
    float g0 = g_mu[om], g1 = g_mu[om + F], g2 = g_mu[om + 2 * F];
    float svw = v0 * w0 + v1 * w1 + v2 * w2;
    float* gs = g_s + a * 3 * F + c;
    gs[0] = gq;
    gs[F] = g0 * w0 + g1 * w1 + g2 * w2;
    gs[2 * F] = gq * svw;
    float gqs3 = gq * s3;
    float* gvw = g_VW + a * 6 * F + c;
    gvw[0] = gqs3 * w0;
    gvw[F] = g0 * s2 + gqs3 * v0;
    gvw[2 * F] = gqs3 * w1;
    gvw[3 * F] = g1 * s2 + gqs3 * v1;
    gvw[4 * F] = gqs3 * w2;
    gvw[5 * F] = g2 * s2 + gqs3 * v2;
}

__global__ void k_mix_ctx_bwd(const float* __restrict__ g_ctx, const float* __restrict__ g_q,
                              const float* __restrict__ VW, int64_t n_atoms, int F, float eps,
                              float* __restrict__ g_q_out, float* __restrict__ g_VW) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F) return;
    int64_t a = t / F;
    int c = (int)(t - a * F);
    const float* v = VW + a * 6 * F + c;
    float v0 = v[0], v1 = v[2 * F], v2 = v[4 * F];
    float n = sqrtf(v0 * v0 + v1 * v1 + v2 * v2 + eps);
    float gn = g_ctx[a * 2 * F + F + c] / n;
    g_q_out[t] = g_q[t] + g_ctx[a * 2 * F + c];
    float* gv = g_VW + a * 6 * F + c;
    gv[0] += gn * v0;
    gv[2 * F] += gn * v1;
    gv[4 * F] += gn * v2;
}

template <int NW, int NRB>
int launch_edge_fwd(const float* x, const float* mu, const float* q, const float* phi, const float* geo,
                    const int* rowptr, const int* slot_j, const float* wf, const float* bf, int n_atoms, int n_edges,
                    int n_rbf, float* q_out, float* mu_out, cudaStream_t st) {
    // exactly one resident wave of CTAs (no tail), >= 32 edges per CTA, at most one CTA per atom
    static int occ_mu = 0, occ_nomu = 0;      // occupancy of a template instantiation: the same on every GPU of a box
    if (!occ_mu) {
        int a = 0, b = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, k_painn_edge_fwd<NW, NRB, true>, NW * 32, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_painn_edge_fwd<NW, NRB, false>, NW * 32, 0);
        occ_nomu = b < 1 ? 1 : b;
        occ_mu = a < 1 ? 1 : a;
    }
    int64_t nb = (int64_t)spk_num_sms() * (mu ? occ_mu : occ_nomu);
    if (nb > spk_cdiv((int64_t)n_edges, 32)) nb = spk_cdiv((int64_t)n_edges, 32);
    if (nb < 1) nb = 1;
    if (nb > n_atoms) nb = n_atoms;
    if (mu)
        spk_launch(k_painn_edge_fwd<NW, NRB, true>, (unsigned)nb, NW * 32, 0, st, x, mu, q, phi, geo, rowptr, slot_j, wf, bf,
                   n_atoms, n_edges, n_rbf, q_out, mu_out);
    else
        spk_launch(k_painn_edge_fwd<NW, NRB, false>, (unsigned)nb, NW * 32, 0, st, x, mu, q, phi, geo, rowptr, slot_j, wf, bf,
                   n_atoms, n_edges, n_rbf, q_out, mu_out);
    return 0;
}

template <int NW, int NRB>
int launch_edge_bwd(const float* x, const float* mu, const float* g_q, const float* g_mu, const float* phi,
                    const float* dphi, const float* geo, const int* sptr, const int* pos_slot, const int* pos_i,
                    const int* slot_eid, const float* wf, const float* bf, int n_atoms, int n_edges, int n_rbf,
                    float* g_x, float* g_mu_in, float* g_rij, int accumulate, cudaStream_t st) {
    static int occ_mu = 0, occ_nomu = 0;
    if (!occ_mu) {
        int a = 0, b = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, k_painn_edge_bwd<NW, NRB, true>, NW * 32, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, k_painn_edge_bwd<NW, NRB, false>, NW * 32, 0);
        occ_nomu = b < 1 ? 1 : b;
        occ_mu = a < 1 ? 1 : a;
    }
    int64_t nb = (int64_t)spk_num_sms() * (mu ? occ_mu : occ_nomu);
    if (nb > spk_cdiv((int64_t)n_edges, 32)) nb = spk_cdiv((int64_t)n_edges, 32);
    if (nb < 1) nb = 1;
    if (nb > n_atoms) nb = n_atoms;
    if (mu)
        spk_launch(k_painn_edge_bwd<NW, NRB, true>, (unsigned)nb, NW * 32, 0, st, x, mu, g_q, g_mu, phi, dphi, geo, sptr,
                   pos_slot, pos_i, slot_eid, wf, bf, n_atoms, n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate);
    else
        spk_launch(k_painn_edge_bwd<NW, NRB, false>, (unsigned)nb, NW * 32, 0, st, x, mu, g_q, g_mu, phi, dphi, geo, sptr,
                   pos_slot, pos_i, slot_eid, wf, bf, n_atoms, n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate);
    return 0;
}

}  // namespace

#define DISPATCH_F_NRB(CALL)                                                   \
    do {                                                                       \
        const int nw_ = F / 32;                                                \
        if (n_rbf <= 20) {                                                     \
            if (nw_ == 1) { CALL(1, 20); } else if (nw_ == 2) { CALL(2, 20); } \
            else if (nw_ == 4) { CALL(4, 20); } else if (nw_ == 8) { CALL(8, 20); } \
            else return SPK_ERR_UNSUPPORTED;                                   \
        } else {                                                               \
            if (nw_ == 1) { CALL(1, 32); } else if (nw_ == 2) { CALL(2, 32); } \
            else if (nw_ == 4) { CALL(4, 32); } else if (nw_ == 8) { CALL(8, 32); } \
            else return SPK_ERR_UNSUPPORTED;                                   \
        }                                                                      \
    } while (0)

extern "C" int spk_painn_edge_fwd(const float* x, const float* mu, const float* q, const float* phi, const float* geo,
                                  const int32_t* rowptr, const int32_t* slot_j, const float* wf, const float* bf,
                                  int64_t n_atoms, int64_t n_edges, int F, int n_rbf, float* q_out, float* mu_out,
                                  spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if ((F & 31) || F > 256 || n_rbf > 32) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !q || !rowptr || !wf || !bf || !q_out || !mu_out) return SPK_ERR_ARG;
    if (n_edges > 0 && (!phi || !geo || !slot_j)) return SPK_ERR_ARG;
    if (mu && mu == mu_out) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
#define CALL_FWD(NW, NRB)                                                                                          \
    launch_edge_fwd<NW, NRB>(x, mu, q, phi, geo, rowptr, slot_j, wf, bf, (int)n_atoms, (int)n_edges, n_rbf, q_out, \
                             mu_out, st)
    DISPATCH_F_NRB(CALL_FWD);
#undef CALL_FWD
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_edge_bwd(const float* x, const float* mu, const float* g_q, const float* g_mu,
                                  const float* phi, const float* dphi, const float* geo, const int32_t* sptr,
                                  const int32_t* pos_slot, const int32_t* pos_i, const int32_t* slot_eid,
                                  const float* wf, const float* bf, int64_t n_atoms, int64_t n_edges, int F, int n_rbf,
                                  float* g_x, float* g_mu_in, float* g_rij, int accumulate, spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if ((F & 31) || F > 256 || n_rbf > 32) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !g_q || !g_mu || !sptr || !wf || !bf || !g_x) return SPK_ERR_ARG;
    if (mu && !g_mu_in) return SPK_ERR_ARG;
    if (n_edges > 0 && (!phi || !dphi || !geo || !pos_slot || !pos_i || !slot_eid || !g_rij)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
#define CALL_BWD(NW, NRB)                                                                                           \
    launch_edge_bwd<NW, NRB>(x, mu, g_q, g_mu, phi, dphi, geo, sptr, pos_slot, pos_i, slot_eid, wf, bf, (int)n_atoms, \
                             (int)n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate, st)
    DISPATCH_F_NRB(CALL_BWD);
#undef CALL_BWD
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

#define GRID1D(n, T) (unsigned)spk_cdiv((n), (T)), (T), 0, spk_st(stream)

extern "C" int spk_painn_mix_ctx(const float* q, const float* VW, int64_t n_atoms, int F, float eps, float* ctx,
                                 spk_stream_t stream) {
    if (n_atoms < 0 || F <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!q || !VW || !ctx) return SPK_ERR_ARG;
    spk_launch(k_mix_ctx, GRID1D(n_atoms * F, 256), q, VW, n_atoms, F, eps, ctx);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_mix_update(const float* q, const float* mu, const float* s, const float* VW, int64_t n_atoms,
                                    int F, float* q_out, float* mu_out, spk_stream_t stream) {
    if (n_atoms < 0 || F <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!q || !mu || !s || !VW || !q_out || !mu_out) return SPK_ERR_ARG;
    spk_launch(k_mix_update, GRID1D(n_atoms * F, 256), q, mu, s, VW, n_atoms, F, q_out, mu_out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_mix_update_bwd(const float* g_q, const float* g_mu, const float* s, const float* VW,
                                        int64_t n_atoms, int F, float* g_s, float* g_VW, spk_stream_t stream) {
    if (n_atoms < 0 || F <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!g_q || !g_mu || !s || !VW || !g_s || !g_VW) return SPK_ERR_ARG;
    spk_launch(k_mix_update_bwd, GRID1D(n_atoms * F, 256), g_q, g_mu, s, VW, n_atoms, F, g_s, g_VW);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_mix_ctx_bwd(const float* g_ctx, const float* g_q, const float* VW, int64_t n_atoms, int F,
                                     float eps, float* g_q_out, float* g_VW, spk_stream_t stream) {
    if (n_atoms < 0 || F <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!g_ctx || !g_q || !VW || !g_q_out || !g_VW) return SPK_ERR_ARG;
    spk_launch(k_mix_ctx_bwd, GRID1D(n_atoms * F, 256), g_ctx, g_q, VW, n_atoms, F, eps, g_q_out, g_VW);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

// Gated equivariant output heads: the GatedEquivariantBlock glue (nn/equivariant.py:57-71) and the DipoleMoment /
// Polarizability heads (atomistic/atomwise.py:172-213, 267-293).
//
// Hidden blocks (n_sin = n_vin = Fi, n_sout = n_vout = Fo): the three Dense layers run on spk_dense_tc / spk_dense; the
// kernels here are the glue around them, thread per (atom, column):
//     ctx   = [s | ||V||]                 VW = mix_vectors(V) [N,3,2Fo], V = VW[..., :Fo], W = VW[..., Fo:]
//     s_out = act(x[:, :Fo]),  v_out = x[:, Fo:] * W        x = scalar_net(ctx) [N,2Fo]
// The norm has no epsilon (torch.norm) and its reverse is 0 where ||V|| = 0, torch's subgradient.
//
// Tail (n_sout = n_vout = 1) + per-system assembly: one CTA of 128 threads takes HT_TILE = 8 consecutive atoms:
// the 2-column vector mix and the norm (warp per atom), the (Fi+1) -> H layer (thread per hidden unit, transposed weight
// read coalesced), the H -> 2 layer (warp per atom), the gate; then the atoms' contributions
//     dipole          [q, q R, R, mu_atomic]          (10 fp64)
//     polarizability  [alpha, nu (x) R]               (10 fp64)
// go through the partial pass of segscan.cuh (seg_partials, which scans a tile of 8 atoms over warp 0 by shuffles), and
// k_head_finish adds each system's CTA partials in a fixed order (bitwise reproducible, no atomics).  With q' = q + c_m, c_m = (Q_m - sum_m q) / n_m the dipole is
//     mu_m = sum q R + c_m sum R + sum mu_atomic,      alpha_m = sum alpha I + S + S^T,  S = sum nu (x) R.
// The reverse kernel recomputes the tail per atom and writes dE/ds, dE/dV and dE/dR directly.
#include "segscan.cuh"

namespace {

constexpr int HT_THREADS = 128;
constexpr int HT_AB = 8;        // atoms per sub-batch of the tail
constexpr int HT_TILE = HT_AB;  // atoms per CTA of the forward (items of the segmented scan): one sub-batch, so that
                                // cfg2's 5376 atoms fill 672 CTAs
constexpr int HT_MAXF = 256;    // Fi and H of the tail
constexpr int HT_NV = 10;
constexpr int HT_SAVED = 8;     // per system: c, R_mean[3], y[3], n

enum { HEAD_DIPOLE = 0, HEAD_POLAR = 1 };

// ------------------------------------------------------------------------------------------------- hidden blocks
__global__ void k_geq_ctx(const float* __restrict__ s, const float* __restrict__ VW, int64_t n_atoms, int Fi, int Fo,
                          float* __restrict__ ctx) {
    SPK_PDL_ENTER();
    const int W = Fi + Fo;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * W) return;
    const int64_t a = t / W;
    const int c = (int)(t - a * W);
    if (c < Fi) {
        ctx[t] = s[a * Fi + c];
        return;
    }
    const float* v = VW + a * 6 * Fo + (c - Fi);
    const float v0 = v[0], v1 = v[2 * Fo], v2 = v[4 * Fo];
    ctx[t] = sqrtf(v0 * v0 + v1 * v1 + v2 * v2);
}

__global__ void k_geq_ctx_bwd(const float* __restrict__ g_ctx, const float* __restrict__ VW, int64_t n_atoms, int Fi,
                              int Fo, float* __restrict__ g_s, float* __restrict__ g_VW) {
    SPK_PDL_ENTER();
    const int W = Fi + Fo;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * W) return;
    const int64_t a = t / W;
    const int c = (int)(t - a * W);
    if (c < Fi) {
        g_s[a * Fi + c] = g_ctx[t];
        return;
    }
    const int64_t o = a * 6 * Fo + (c - Fi);
    const float v0 = VW[o], v1 = VW[o + 2 * Fo], v2 = VW[o + 4 * Fo];
    const float n = sqrtf(v0 * v0 + v1 * v1 + v2 * v2);
    const float g = n > 0.f ? g_ctx[t] / n : 0.f;
    g_VW[o] = g * v0;
    g_VW[o + 2 * Fo] = g * v1;
    g_VW[o + 4 * Fo] = g * v2;
}

__global__ void k_geq_gate(const float* __restrict__ x, const float* __restrict__ VW, int64_t n_atoms, int Fo, int act,
                           float* __restrict__ s_out, float* __restrict__ v_out) {
    SPK_PDL_ENTER();
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * Fo) return;
    const int64_t a = t / Fo;
    const int c = (int)(t - a * Fo);
    s_out[t] = spk_act(x[a * 2 * Fo + c], act);
    const float xv = x[a * 2 * Fo + Fo + c];
    const float* w = VW + a * 6 * Fo + Fo + c;
    float* v = v_out + a * 3 * Fo + c;
    v[0] = xv * w[0];
    v[Fo] = xv * w[2 * Fo];
    v[2 * Fo] = xv * w[4 * Fo];
}

__global__ void k_geq_gate_bwd(const float* __restrict__ g_s, const float* __restrict__ g_v, const float* __restrict__ x,
                               const float* __restrict__ VW, int64_t n_atoms, int Fo, int act, float* __restrict__ g_x,
                               float* __restrict__ g_VW) {
    SPK_PDL_ENTER();
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * Fo) return;
    const int64_t a = t / Fo;
    const int c = (int)(t - a * Fo);
    const float* xa = x + a * 2 * Fo;
    g_x[a * 2 * Fo + c] = g_s ? g_s[t] * spk_act_grad(xa[c], act) : 0.f;
    const float xv = xa[Fo + c];
    const int64_t o = a * 6 * Fo + Fo + c;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (g_v) {
        const float* gv = g_v + a * 3 * Fo + c;
        g0 = gv[0], g1 = gv[Fo], g2 = gv[2 * Fo];
    }
    g_x[a * 2 * Fo + Fo + c] = g0 * VW[o] + g1 * VW[o + 2 * Fo] + g2 * VW[o + 4 * Fo];
    g_VW[o] = g0 * xv;
    g_VW[o + 2 * Fo] = g1 * xv;
    g_VW[o + 4 * Fo] = g2 * xv;
}

// ------------------------------------------------------------------------------------------------- tail
struct TailW {
    const float* wmix;   // [2, Fi]      mix_vectors.weight
    const float* w0;     // [H, Fi+1]    scalar_net.0.weight
    const float* w0t;    // [Fi+1, H]    its transpose
    const float* b0;     // [H]
    const float* w1;     // [2, H]       scalar_net.1.weight
    const float* b1;     // [2]
    int Fi, H, act;
};

struct TailSmem {
    float ctx[HT_AB][HT_MAXF + 1];
    float h[HT_AB][HT_MAXF];      // act(pre); the reverse keeps act'(pre) in hd
    float hd[HT_AB][HT_MAXF];
    float vm[HT_AB][6];           // [c][d]: mixed vector column c (0 = V, 1 = W), component d
    float o[HT_AB][2];            // scalar_net output (charge / alpha, gate)
};

// Forward of the tail for atoms a0 .. a0 + HT_AB - 1 (< n_atoms); leaves vm, ctx, h (+ hd if need_d) and o in shared memory.
__device__ __forceinline__ void tail_eval(const float* __restrict__ s, const float* __restrict__ V, int64_t a0,
                                          int64_t n_atoms, const TailW& w, TailSmem& sm, bool need_d) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int Fi = w.Fi, H = w.H;
    for (int r = warp; r < HT_AB; r += HT_THREADS / 32) {
        const int64_t a = a0 + r;
        float p[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (a < n_atoms) {
            for (int k = lane; k < Fi; k += 32) {
                const float m0 = w.wmix[k], m1 = w.wmix[Fi + k];
                const float* v = V + a * 3 * Fi + k;
                const float x0 = v[0], x1 = v[Fi], x2 = v[2 * Fi];
                p[0] = fmaf(m0, x0, p[0]); p[1] = fmaf(m0, x1, p[1]); p[2] = fmaf(m0, x2, p[2]);
                p[3] = fmaf(m1, x0, p[3]); p[4] = fmaf(m1, x1, p[4]); p[5] = fmaf(m1, x2, p[5]);
                sm.ctx[r][k] = s[a * Fi + k];
            }
        } else {
            for (int k = lane; k < Fi; k += 32) sm.ctx[r][k] = 0.f;
        }
#pragma unroll
        for (int c = 0; c < 6; ++c) p[c] = spk_warp_sum(p[c]);
        if (lane == 0) {
#pragma unroll
            for (int c = 0; c < 6; ++c) sm.vm[r][c] = p[c];
            sm.ctx[r][Fi] = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
        }
    }
    __syncthreads();
    for (int j = t; j < H; j += HT_THREADS) {
        float acc[HT_AB];
        const float bj = w.b0[j];
#pragma unroll
        for (int r = 0; r < HT_AB; ++r) acc[r] = bj;
        for (int k = 0; k <= Fi; ++k) {
            const float wk = w.w0t[(int64_t)k * H + j];
#pragma unroll
            for (int r = 0; r < HT_AB; ++r) acc[r] = fmaf(wk, sm.ctx[r][k], acc[r]);
        }
#pragma unroll
        for (int r = 0; r < HT_AB; ++r) {
            if (need_d) {
                spk_act_both(acc[r], w.act, sm.h[r][j], sm.hd[r][j]);
            } else {
                sm.h[r][j] = spk_act(acc[r], w.act);
            }
        }
    }
    __syncthreads();
    for (int r = warp; r < HT_AB; r += HT_THREADS / 32) {
        float o0 = 0.f, o1 = 0.f;
        for (int j = lane; j < H; j += 32) {
            o0 = fmaf(w.w1[j], sm.h[r][j], o0);
            o1 = fmaf(w.w1[H + j], sm.h[r][j], o1);
        }
        o0 = spk_warp_sum(o0);
        o1 = spk_warp_sum(o1);
        if (lane == 0) {
            sm.o[r][0] = o0 + w.b1[0];
            sm.o[r][1] = o1 + w.b1[1];
        }
    }
    __syncthreads();
}

__device__ __forceinline__ void atom_terms(int mode, float q, const float* nu, const float* R, double (&v)[HT_NV]) {
    const double rx = R[0], ry = R[1], rz = R[2];
    v[0] = q;
    if (mode == HEAD_DIPOLE) {
        v[1] = (double)q * rx; v[2] = (double)q * ry; v[3] = (double)q * rz;
        v[4] = rx; v[5] = ry; v[6] = rz;
        v[7] = nu[0]; v[8] = nu[1]; v[9] = nu[2];
    } else {
        const double r[3] = {rx, ry, rz};
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) v[1 + 3 * i + j] = (double)nu[i] * r[j];
    }
}

template <int MODE>
__global__ void __launch_bounds__(HT_THREADS) k_head_tail(const float* __restrict__ s, const float* __restrict__ V,
                                                          const float* __restrict__ R, const int64_t* __restrict__ idx_m,
                                                          const int32_t* __restrict__ sys_ptr, int64_t n_atoms, TailW w,
                                                          float* __restrict__ q_atom, double* __restrict__ sys_part,
                                                          double* __restrict__ head) {
    static_assert(HT_TILE <= 32, "the tail's partials use the warp scan");
    __shared__ TailSmem sm;
    __shared__ float res[HT_TILE][4];
    SPK_PDL_ENTER();
    const int64_t b0 = (int64_t)blockIdx.x * HT_TILE;
    for (int sb = 0; sb < HT_TILE; sb += HT_AB) {
        if (b0 + sb >= n_atoms) break;
        tail_eval(s, V, b0 + sb, n_atoms, w, sm, false);
        if (threadIdx.x < HT_AB) {
            const int r = threadIdx.x;
            res[sb + r][0] = sm.o[r][0];
#pragma unroll
            for (int d = 0; d < 3; ++d) res[sb + r][1 + d] = sm.o[r][1] * sm.vm[r][3 + d];
        }
        __syncthreads();   // sm is rewritten by the next sub-batch
    }
    const int t = threadIdx.x;
    const int64_t a = b0 + t;
    double v[HT_NV];
#pragma unroll
    for (int c = 0; c < HT_NV; ++c) v[c] = 0.0;
    int64_t m = 0, first = 0, end = 0;
    if (t < HT_TILE && a < n_atoms) {
        atom_terms(MODE, res[t][0], &res[t][1], R + 3 * a, v);
        if (q_atom) q_atom[a] = res[t][0];
        m = idx_m[a];
        first = sys_ptr[m];
        end = sys_ptr[m + 1];
    }
    if (threadIdx.x >= 32) return;
    seg_partials<HT_TILE, HT_NV>(v, n_atoms, m, first, end, sys_part, head);
}

// charges from the scalar MLP (use_vector_representation=False): the same assembly without atomic dipoles
constexpr int HS_TILE = HT_THREADS;

__global__ void __launch_bounds__(HT_THREADS) k_head_scalar(const float* __restrict__ q, const float* __restrict__ R,
                                                            const int64_t* __restrict__ idx_m,
                                                            const int32_t* __restrict__ sys_ptr, int64_t n_atoms,
                                                            double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * HS_TILE + threadIdx.x;
    double v[HT_NV];
#pragma unroll
    for (int c = 0; c < HT_NV; ++c) v[c] = 0.0;
    int64_t m = 0, first = 0, end = 0;
    if (a < n_atoms) {
        const float zero[3] = {0.f, 0.f, 0.f};
        atom_terms(HEAD_DIPOLE, q[a], zero, R + 3 * a, v);
        m = idx_m[a];
        first = sys_ptr[m];
        end = sys_ptr[m + 1];
    }
    seg_partials<HS_TILE, HT_NV>(v, n_atoms, m, first, end, sys_part, head);
}

// Per system: the totals, the outputs and what the reverse needs (saved[m] = c, R_mean, y, n).
template <int MODE, int TILE>
__global__ void __launch_bounds__(SEG_FIN_T) k_head_finish(const int32_t* __restrict__ sys_ptr,
                                                           const double* __restrict__ sys_part,
                                                           const double* __restrict__ head,
                                                           const float* __restrict__ total_charge, int correct,
                                                           int magnitude, float* __restrict__ out,
                                                           double* __restrict__ saved) {
    __shared__ double red[HT_NV][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t m = blockIdx.x;
    seg_finish_block<TILE, HT_NV>(sys_ptr, nullptr, sys_part, head, m, red);
    if (threadIdx.x != 0) return;
    double tot[HT_NV];
#pragma unroll
    for (int c = 0; c < HT_NV; ++c) tot[c] = red[c][0];
    const int64_t n = sys_ptr[m + 1] - sys_ptr[m];
    double* sv = saved + m * HT_SAVED;
    if (MODE == HEAD_DIPOLE) {
        double c = 0.0;
        if (correct && n > 0) c = ((total_charge ? (double)total_charge[m] : 0.0) - tot[0]) / (double)n;
        double y[3];
        for (int d = 0; d < 3; ++d) {
            y[d] = tot[1 + d] + c * tot[4 + d] + tot[7 + d];
            sv[1 + d] = n > 0 ? tot[4 + d] / (double)n : 0.0;
            sv[4 + d] = y[d];
        }
        sv[0] = c;
        sv[7] = (double)n;
        if (magnitude) {
            out[m] = (float)sqrt(y[0] * y[0] + y[1] * y[1] + y[2] * y[2]);
        } else {
            for (int d = 0; d < 3; ++d) out[m * 3 + d] = (float)y[d];
        }
    } else {
        for (int c = 0; c < HT_SAVED; ++c) sv[c] = 0.0;   // nothing of the polarizability's reverse is saved
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j)
                out[m * 9 + 3 * i + j] = (float)((i == j ? tot[0] : 0.0) + tot[1 + 3 * i + j] + tot[1 + 3 * j + i]);
    }
}

__global__ void k_head_charges(const float* __restrict__ q_atom, const int64_t* __restrict__ idx_m,
                               const double* __restrict__ saved, int64_t n_atoms, float* __restrict__ charges) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    charges[a] = (float)((double)q_atom[a] + saved[idx_m[a] * HT_SAVED]);
}

// The per-system output gradient seen by one atom: dipole -> (g_q, g_mu, g_R); polarizability -> (g_alpha, g_nu, g_R).
// ``nu`` (atomic dipole / anisotropic vector) and ``q`` are the atom's tail outputs.
__device__ __forceinline__ void head_atom_grad(int mode, const float* __restrict__ g_out, const double* __restrict__ sv,
                                               int correct, int magnitude, float q, const float* nu, const float* R,
                                               float& g_q, float* g_nu, float* g_R) {
    if (mode == HEAD_DIPOLE) {
        double g[3];
        if (magnitude) {
            const double y0 = sv[4], y1 = sv[5], y2 = sv[6];
            const double ny = sqrt(y0 * y0 + y1 * y1 + y2 * y2);
            const double f = ny > 0.0 ? (double)g_out[0] / ny : 0.0;
            g[0] = f * y0, g[1] = f * y1, g[2] = f * y2;
        } else {
            g[0] = g_out[0], g[1] = g_out[1], g[2] = g_out[2];
        }
        double gq = 0.0;
        const double qp = (double)q + sv[0];
        for (int d = 0; d < 3; ++d) {
            gq += g[d] * ((double)R[d] - (correct ? sv[1 + d] : 0.0));
            g_nu[d] = (float)g[d];
            g_R[d] = (float)(g[d] * qp);
        }
        g_q = (float)gq;
    } else {
        float Gs[3][3];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) Gs[i][j] = g_out[3 * i + j] + g_out[3 * j + i];
        g_q = g_out[0] + g_out[4] + g_out[8];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            g_nu[i] = Gs[i][0] * R[0] + Gs[i][1] * R[1] + Gs[i][2] * R[2];
            g_R[i] = Gs[0][i] * nu[0] + Gs[1][i] * nu[1] + Gs[2][i] * nu[2];
        }
    }
}

template <int MODE>
__global__ void __launch_bounds__(HT_THREADS) k_head_tail_bwd(
    const float* __restrict__ s, const float* __restrict__ V, const float* __restrict__ R,
    const int64_t* __restrict__ idx_m, const double* __restrict__ saved, const float* __restrict__ g_out,
    const float* __restrict__ g_qx, int correct, int magnitude, int64_t n_atoms, TailW w, float* __restrict__ g_s,
    float* __restrict__ g_V, float* __restrict__ g_R) {
    __shared__ TailSmem sm;
    __shared__ float go[HT_AB][2];
    __shared__ float gvm[HT_AB][6];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int Fi = w.Fi, H = w.H;
    const int64_t a0 = (int64_t)blockIdx.x * HT_AB;
    tail_eval(s, V, a0, n_atoms, w, sm, true);
    if (t < HT_AB) {
        const int r = t;
        const int64_t a = a0 + r;
        float gq = 0.f, gnu[3] = {0.f, 0.f, 0.f}, gR[3];
        if (a < n_atoms) {
            const int64_t m = idx_m[a];
            const int no = MODE == HEAD_DIPOLE ? (magnitude ? 1 : 3) : 9;
            const float nu[3] = {sm.o[r][1] * sm.vm[r][3], sm.o[r][1] * sm.vm[r][4], sm.o[r][1] * sm.vm[r][5]};
            head_atom_grad(MODE, g_out + m * no, saved + m * HT_SAVED, correct, magnitude, sm.o[r][0], nu, R + 3 * a, gq,
                           gnu, gR);
            if (g_qx) gq += g_qx[a];     // gradient of the charges output (spk_head_bwd_q)
            for (int d = 0; d < 3; ++d) g_R[3 * a + d] = gR[d];
        }
        // nu = o1 * vm1  ->  g_o1 = g_nu . vm1,  g_vm1 = g_nu * o1
        go[r][0] = gq;
        go[r][1] = gnu[0] * sm.vm[r][3] + gnu[1] * sm.vm[r][4] + gnu[2] * sm.vm[r][5];
        for (int d = 0; d < 3; ++d) gvm[r][3 + d] = gnu[d] * sm.o[r][1];
    }
    __syncthreads();
    for (int j = t; j < H; j += HT_THREADS) {
        const float w10 = w.w1[j], w11 = w.w1[H + j];
#pragma unroll
        for (int r = 0; r < HT_AB; ++r) sm.h[r][j] = (w10 * go[r][0] + w11 * go[r][1]) * sm.hd[r][j];
    }
    __syncthreads();
    for (int k = t; k <= Fi; k += HT_THREADS) {
        float acc[HT_AB];
#pragma unroll
        for (int r = 0; r < HT_AB; ++r) acc[r] = 0.f;
        for (int j = 0; j < H; ++j) {
            const float wj = w.w0[(int64_t)j * (Fi + 1) + k];
#pragma unroll
            for (int r = 0; r < HT_AB; ++r) acc[r] = fmaf(wj, sm.h[r][j], acc[r]);
        }
#pragma unroll
        for (int r = 0; r < HT_AB; ++r) {
            const int64_t a = a0 + r;
            if (k < Fi) {
                if (a < n_atoms) g_s[a * Fi + k] = acc[r];
            } else {
                const float n = sm.ctx[r][Fi];
                const float g = n > 0.f ? acc[r] / n : 0.f;
                for (int d = 0; d < 3; ++d) gvm[r][d] = g * sm.vm[r][d];
            }
        }
    }
    __syncthreads();
    for (int k = t; k < Fi; k += HT_THREADS) {
        const float m0 = w.wmix[k], m1 = w.wmix[Fi + k];
#pragma unroll
        for (int r = 0; r < HT_AB; ++r) {
            const int64_t a = a0 + r;
            if (a >= n_atoms) break;
            float* gv = g_V + a * 3 * Fi + k;
            gv[0] = m0 * gvm[r][0] + m1 * gvm[r][3];
            gv[Fi] = m0 * gvm[r][1] + m1 * gvm[r][4];
            gv[2 * Fi] = m0 * gvm[r][2] + m1 * gvm[r][5];
        }
    }
}

// reverse of the scalar-charge assembly: g_hid = g_q (x) w1 (the last Dense H -> 1) and g_R, thread per (atom, hidden unit)
__global__ void k_head_scalar_bwd(const float* __restrict__ q, const float* __restrict__ R,
                                  const int64_t* __restrict__ idx_m, const double* __restrict__ saved,
                                  const float* __restrict__ g_out, const float* __restrict__ g_qx, int correct,
                                  int magnitude, const float* __restrict__ w1, int64_t n_atoms, int H,
                                  float* __restrict__ g_hid, float* __restrict__ g_R) {
    SPK_PDL_ENTER();
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * H) return;
    const int64_t a = t / H;
    const int j = (int)(t - a * H);
    const int64_t m = idx_m[a];
    float gq, gnu[3], gR[3];
    const float zero[3] = {0.f, 0.f, 0.f};
    head_atom_grad(HEAD_DIPOLE, g_out + m * (magnitude ? 1 : 3), saved + m * HT_SAVED, correct, magnitude, q[a], zero,
                   R + 3 * a, gq, gnu, gR);
    if (g_qx) gq += g_qx[a];             // gradient of the charges output (spk_head_scalar_bwd_q)
    g_hid[t] = gq * w1[j];
    if (j == 0)
        for (int d = 0; d < 3; ++d) g_R[3 * a + d] = gR[d];
}

// Reverse of the charge correction q' = q + (Q_m - sum_m q) / n_m: g_q = g_q' - mean_m(g_q').  The per-system sums of g_q'
// run through the segmented-partial pass of segscan.cuh (CTAs of HC_T atoms), so they are bitwise reproducible.
constexpr int HC_T = 256;

__global__ void __launch_bounds__(HC_T) k_charges_bwd_partials(const float* __restrict__ g_c,
                                                               const int64_t* __restrict__ idx_m,
                                                               const int32_t* __restrict__ sys_ptr, int64_t n_atoms,
                                                               double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * HC_T + threadIdx.x;
    double v[1] = {0.0};
    int64_t m = 0, first = 0, end = 0;
    if (a < n_atoms) {
        v[0] = g_c[a];
        m = idx_m[a];
        first = sys_ptr[m];
        end = sys_ptr[m + 1];
    }
    seg_partials<HC_T, 1>(v, n_atoms, m, first, end, sys_part, head);
}

__global__ void __launch_bounds__(SEG_FIN_T) k_charges_bwd_mean(const int32_t* __restrict__ sys_ptr,
                                                                const double* __restrict__ sys_part,
                                                                const double* __restrict__ head,
                                                                double* __restrict__ mean) {
    __shared__ double red[1][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t m = blockIdx.x;
    seg_finish_block<HC_T, 1>(sys_ptr, nullptr, sys_part, head, m, red);
    if (threadIdx.x != 0) return;
    const int64_t n = sys_ptr[m + 1] - sys_ptr[m];
    mean[m] = n > 0 ? red[0][0] / (double)n : 0.0;
}

__global__ void k_charges_bwd_apply(const float* __restrict__ g_c, const int64_t* __restrict__ idx_m,
                                    const double* __restrict__ mean, int64_t n_atoms, float* __restrict__ g_q) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    g_q[a] = mean ? (float)((double)g_c[a] - mean[idx_m[a]]) : g_c[a];
}

}  // namespace

#define GRID1D(n, T) (unsigned)spk_cdiv((n), (T)), (T), 0, spk_st(stream)

extern "C" int spk_geq_ctx(const float* s, const float* VW, int64_t n_atoms, int Fi, int Fo, float* ctx,
                           spk_stream_t stream) {
    if (n_atoms < 0 || Fi <= 0 || Fo <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!s || !VW || !ctx) return SPK_ERR_ARG;
    spk_launch(k_geq_ctx, GRID1D(n_atoms * (Fi + Fo), 256), s, VW, n_atoms, Fi, Fo, ctx);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_geq_ctx_bwd(const float* g_ctx, const float* VW, int64_t n_atoms, int Fi, int Fo, float* g_s,
                               float* g_VW, spk_stream_t stream) {
    if (n_atoms < 0 || Fi <= 0 || Fo <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!g_ctx || !VW || !g_s || !g_VW) return SPK_ERR_ARG;
    spk_launch(k_geq_ctx_bwd, GRID1D(n_atoms * (Fi + Fo), 256), g_ctx, VW, n_atoms, Fi, Fo, g_s, g_VW);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_geq_gate(const float* x, const float* VW, int64_t n_atoms, int Fo, int act, float* s_out,
                            float* v_out, spk_stream_t stream) {
    if (n_atoms < 0 || Fo <= 0 || act < 0 || act > 2) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !VW || !s_out || !v_out) return SPK_ERR_ARG;
    spk_launch(k_geq_gate, GRID1D(n_atoms * Fo, 256), x, VW, n_atoms, Fo, act, s_out, v_out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_geq_gate_bwd(const float* g_s, const float* g_v, const float* x, const float* VW, int64_t n_atoms,
                                int Fo, int act, float* g_x, float* g_VW, spk_stream_t stream) {
    if (n_atoms < 0 || Fo <= 0 || act < 0 || act > 2) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!x || !VW || !g_x || !g_VW) return SPK_ERR_ARG;
    spk_launch(k_geq_gate_bwd, GRID1D(n_atoms * Fo, 256), g_s, g_v, x, VW, n_atoms, Fo, act, g_x, g_VW);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" size_t spk_head_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? spk_cdiv(n_atoms, HT_TILE) : 0;
    return sizeof(double) * (size_t)(HT_NV * ((n_sys > 0 ? n_sys : 0) + nb + 1));
}

static int check_tail(const spk_head_tail_t* w) {
    if (!w || w->Fi <= 0 || w->H <= 0 || w->act < 0 || w->act > 2) return SPK_ERR_ARG;
    if (w->Fi > HT_MAXF || w->H > HT_MAXF) return SPK_ERR_UNSUPPORTED;
    if (!w->wmix || !w->w0 || !w->w0t || !w->b0 || !w->w1 || !w->b1) return SPK_ERR_ARG;
    return SPK_OK;
}

static TailW tail_of(const spk_head_tail_t* w) {
    return TailW{w->wmix, w->w0, w->w0t, w->b0, w->w1, w->b1, w->Fi, w->H, w->act};
}

extern "C" int spk_head_fwd(int kind, const spk_head_tail_t* tail, const float* s, const float* V, const float* q,
                            const float* R, const int64_t* idx_m, const int32_t* sys_ptr, const float* total_charge,
                            int64_t n_atoms, int64_t n_sys, int correct, int magnitude, float* out, float* q_atom,
                            double* saved, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (n_atoms < 0 || n_sys < 0 || n_atoms >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (kind != SPK_HEAD_DIPOLE && kind != SPK_HEAD_POLAR) return SPK_ERR_ARG;
    if (n_sys == 0) return SPK_OK;
    if (!sys_ptr || !out || !saved || !workspace) return SPK_ERR_ARG;
    if (workspace_bytes < spk_head_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!R || !idx_m)) return SPK_ERR_ARG;
    if (kind == SPK_HEAD_POLAR && (!tail || magnitude)) return SPK_ERR_ARG;
    if (tail) {
        const int rc = check_tail(tail);
        if (rc != SPK_OK) return rc;
        if (n_atoms > 0 && (!s || !V)) return SPK_ERR_ARG;
    } else if (n_atoms > 0 && !q) {
        return SPK_ERR_ARG;
    }
    double* sys_part = reinterpret_cast<double*>(workspace);
    double* head = sys_part + HT_NV * n_sys;
    const cudaStream_t st = spk_st(stream);
    if (tail) {
        const TailW w = tail_of(tail);
        if (n_atoms > 0) {
            if (kind == SPK_HEAD_DIPOLE)
                spk_launch(k_head_tail<HEAD_DIPOLE>, (unsigned)spk_cdiv(n_atoms, HT_TILE), HT_THREADS, 0, st, s, V, R,
                           idx_m, sys_ptr, n_atoms, w, q_atom, sys_part, head);
            else
                spk_launch(k_head_tail<HEAD_POLAR>, (unsigned)spk_cdiv(n_atoms, HT_TILE), HT_THREADS, 0, st, s, V, R,
                           idx_m, sys_ptr, n_atoms, w, q_atom, sys_part, head);
        }
        if (kind == SPK_HEAD_DIPOLE)
            spk_launch(k_head_finish<HEAD_DIPOLE, HT_TILE>, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, sys_part, head,
                       total_charge, correct, magnitude, out, saved);
        else
            spk_launch(k_head_finish<HEAD_POLAR, HT_TILE>, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, sys_part, head,
                       total_charge, correct, magnitude, out, saved);
    } else {
        if (n_atoms > 0)
            spk_launch(k_head_scalar, (unsigned)spk_cdiv(n_atoms, HS_TILE), HT_THREADS, 0, st, q, R, idx_m, sys_ptr,
                       n_atoms, sys_part, head);
        spk_launch(k_head_finish<HEAD_DIPOLE, HS_TILE>, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, sys_part, head,
                   total_charge, correct, magnitude, out, saved);
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_head_charges(const float* q_atom, const int64_t* idx_m, const double* saved, int64_t n_atoms,
                                float* charges, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!q_atom || !idx_m || !saved || !charges) return SPK_ERR_ARG;
    spk_launch(k_head_charges, GRID1D(n_atoms, 256), q_atom, idx_m, saved, n_atoms, charges);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_head_bwd(int kind, const spk_head_tail_t* tail, const float* s, const float* V, const float* R,
                            const int64_t* idx_m, const double* saved, const float* g_out, int64_t n_atoms, int correct,
                            int magnitude, float* g_s, float* g_V, float* g_R, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (kind != SPK_HEAD_DIPOLE && kind != SPK_HEAD_POLAR) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    const int rc = check_tail(tail);
    if (rc != SPK_OK) return rc;
    if (!s || !V || !R || !idx_m || !saved || !g_out || !g_s || !g_V || !g_R) return SPK_ERR_ARG;
    if (kind == SPK_HEAD_POLAR && magnitude) return SPK_ERR_ARG;
    const TailW w = tail_of(tail);
    const unsigned nb = (unsigned)spk_cdiv(n_atoms, HT_AB);
    if (kind == SPK_HEAD_DIPOLE)
        spk_launch(k_head_tail_bwd<HEAD_DIPOLE>, nb, HT_THREADS, 0, spk_st(stream), s, V, R, idx_m, saved, g_out,
                   (const float*)nullptr, correct, magnitude, n_atoms, w, g_s, g_V, g_R);
    else
        spk_launch(k_head_tail_bwd<HEAD_POLAR>, nb, HT_THREADS, 0, spk_st(stream), s, V, R, idx_m, saved, g_out,
                   (const float*)nullptr, correct, magnitude, n_atoms, w, g_s, g_V, g_R);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_head_scalar_bwd(const float* q, const float* R, const int64_t* idx_m, const double* saved,
                                   const float* g_out, int correct, int magnitude, const float* w1, int64_t n_atoms, int H,
                                   float* g_hid, float* g_R, spk_stream_t stream) {
    if (n_atoms < 0 || H <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!q || !R || !idx_m || !saved || !g_out || !w1 || !g_hid || !g_R) return SPK_ERR_ARG;
    spk_launch(k_head_scalar_bwd, GRID1D(n_atoms * H, 256), q, R, idx_m, saved, g_out, (const float*)nullptr, correct,
               magnitude, w1, n_atoms, H, g_hid, g_R);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" size_t spk_head_charges_bwd_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? spk_cdiv(n_atoms, HC_T) : 0;
    const int64_t B = n_sys > 0 ? n_sys : 0;
    return sizeof(double) * (size_t)(2 * B + nb + 1);
}

extern "C" int spk_head_charges_bwd(const float* g_charges, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                                    int64_t n_sys, int correct, float* g_q, void* workspace, size_t workspace_bytes,
                                    spk_stream_t stream) {
    if (n_atoms < 0 || n_sys < 0 || n_atoms >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!g_charges || !idx_m || !g_q) return SPK_ERR_ARG;
    const cudaStream_t st = spk_st(stream);
    double* mean = nullptr;
    if (correct && n_sys > 0) {
        if (!sys_ptr || !workspace || workspace_bytes < spk_head_charges_bwd_workspace_bytes(n_atoms, n_sys))
            return SPK_ERR_ARG;
        mean = reinterpret_cast<double*>(workspace);
        double* sys_part = mean + n_sys;
        double* head = sys_part + n_sys;
        spk_launch(k_charges_bwd_partials, (unsigned)spk_cdiv(n_atoms, HC_T), HC_T, 0, st, g_charges, idx_m, sys_ptr,
                   n_atoms, sys_part, head);
        spk_launch(k_charges_bwd_mean, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, (const double*)sys_part,
                   (const double*)head, mean);
    }
    spk_launch(k_charges_bwd_apply, GRID1D(n_atoms, 256), g_charges, idx_m, (const double*)mean, n_atoms, g_q);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_head_bwd_q(int kind, const spk_head_tail_t* tail, const float* s, const float* V, const float* R,
                              const int64_t* idx_m, const double* saved, const float* g_out, const float* g_q,
                              int64_t n_atoms, int correct, int magnitude, float* g_s, float* g_V, float* g_R,
                              spk_stream_t stream) {
    if (n_atoms < 0 || kind != SPK_HEAD_DIPOLE) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    const int rc = check_tail(tail);
    if (rc != SPK_OK) return rc;
    if (!s || !V || !R || !idx_m || !saved || !g_out || !g_q || !g_s || !g_V || !g_R) return SPK_ERR_ARG;
    spk_launch(k_head_tail_bwd<HEAD_DIPOLE>, (unsigned)spk_cdiv(n_atoms, HT_AB), HT_THREADS, 0, spk_st(stream), s, V, R,
               idx_m, saved, g_out, g_q, correct, magnitude, n_atoms, tail_of(tail), g_s, g_V, g_R);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_head_scalar_bwd_q(const float* q, const float* R, const int64_t* idx_m, const double* saved,
                                     const float* g_out, const float* g_q, int correct, int magnitude, const float* w1,
                                     int64_t n_atoms, int H, float* g_hid, float* g_R, spk_stream_t stream) {
    if (n_atoms < 0 || H <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!q || !R || !idx_m || !saved || !g_out || !g_q || !w1 || !g_hid || !g_R) return SPK_ERR_ARG;
    spk_launch(k_head_scalar_bwd, GRID1D(n_atoms * H, 256), q, R, idx_m, saved, g_out, g_q, correct, magnitude, w1,
               n_atoms, H, g_hid, g_R);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

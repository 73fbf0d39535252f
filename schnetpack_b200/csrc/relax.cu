// Batchwise L-BFGS relaxation on the device (interfaces/batchwise_optimization.py:613-917, ASEBatchwiseLBFGS.step and
// determine_step), one independent optimizer per system of a collated batch, all state fp64.
//
// The two-loop recursion is a chain of 2 L dependent dot products per system (L = min(memory, iteration)), so a step
// costs reduction latency, not bandwidth.  Two kernels share the same step and differ in who owns a system:
//   * k_lbfgs_warp: one warp per system of at most SPK_RELAX_WARP_ATOMS atoms; every lane keeps the direction of its
//     atoms in registers, dot products are shuffle sums;
//   * k_lbfgs_cluster: a thread-block cluster of RELAX_CL_CTAS CTAs per larger system; the direction lives in the
//     caller's p buffer (each thread only touches its own atoms), dot products are CTA sums exchanged through
//     distributed shared memory, added by every CTA in rank order.
// Every sum has a fixed order given the layout, so a replay is bitwise reproducible; there are no atomics.
#include <cooperative_groups.h>

#include "relax_common.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int WARP_KA = SPK_RELAX_WARP_ATOMS / 32;   // atoms per lane of the warp path
constexpr int WARP_CTA_WARPS = 4;
constexpr int RELAX_CL_CTAS = 8;                     // portable cluster size
constexpr int RELAX_CL_T = 512;
constexpr int CONV_WARPS = 8;

__device__ __forceinline__ double warp_sum_d(double v) {
    // xor butterfly: every lane adds the same two partial sums (in commuted order) at every level, so all lanes end
    // with the bitwise same total
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---- warp per system -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(WARP_CTA_WARPS * 32) k_lbfgs_warp(spk_lbfgs_t st, const float* __restrict__ forces) {
    extern __shared__ double alpha_sm[];                 // [WARP_CTA_WARPS][memory]
    SPK_PDL_ENTER();
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const int64_t w = (int64_t)blockIdx.x * WARP_CTA_WARPS + wib;
    const int64_t it = st.counter[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) st.counter[1] = it + 1;
    if (w >= st.n_warp) return;
    double* alpha = alpha_sm + (int64_t)wib * st.memory;
    const int64_t m = st.order[w];
    const int64_t a0 = st.sys_ptr[m];
    const int n = st.sys_ptr[m + 1] - (int)a0;
    const int64_t D = 3 * st.n_atoms;
    const int64_t M = st.memory;
    const int64_t ns = st.n_sys;

    double q[3 * WARP_KA];
    // 1. history entry of the previous step (update, :886-909) and q = -f
    double ys = 0.0;
#pragma unroll
    for (int k = 0; k < WARP_KA; ++k) {
        const int la = lane + 32 * k;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            q[3 * k + c] = 0.0;
            if (la < n) {
                const int64_t e = 3 * (a0 + la) + c;
                const double f =
                    optimizer_force(st.fixed && st.fixed[a0 + la], forces, st.force_conversion, a0 + la, c);
                if (it > 0) {
                    const int64_t sl = (it - 1) % M;
                    const double s = st.r[e] - st.r0[e];
                    const double y = st.f0[e] - f;
                    st.s[sl * D + e] = s;
                    st.y[sl * D + e] = y;
                    ys += y * s;
                }
                q[3 * k + c] = -f;
            }
        }
    }
    if (it > 0) {
        ys = warp_sum_d(ys);
        if (lane == 0) st.rho[((it - 1) % M) * ns + m] = ys > 1e-8 ? 1.0 / ys : 1.0;
        __syncwarp();
    }
    // 2. two-loop recursion over the last L entries, oldest first; entry i is ring slot (it - L + i) % M
    const int64_t L = it < M ? it : M;
    for (int64_t i = L - 1; i >= 0; --i) {
        const int64_t sl = (it - L + i) % M;
        const double* si = st.s + sl * D + 3 * a0;
        const double* yi = st.y + sl * D + 3 * a0;
        double part = 0.0;
#pragma unroll
        for (int k = 0; k < WARP_KA; ++k) {
            const int la = lane + 32 * k;
            if (la < n) {
#pragma unroll
                for (int c = 0; c < 3; ++c) part += si[3 * la + c] * q[3 * k + c];
            }
        }
        const double a = st.rho[sl * ns + m] * warp_sum_d(part);
        if (lane == 0) alpha[i] = a;
#pragma unroll
        for (int k = 0; k < WARP_KA; ++k) {
            const int la = lane + 32 * k;
            if (la < n) {
#pragma unroll
                for (int c = 0; c < 3; ++c) q[3 * k + c] -= a * yi[3 * la + c];
            }
        }
    }
    __syncwarp();
#pragma unroll
    for (int j = 0; j < 3 * WARP_KA; ++j) q[j] *= st.h0;      // z = H0 q
    for (int64_t i = 0; i < L; ++i) {
        const int64_t sl = (it - L + i) % M;
        const double* si = st.s + sl * D + 3 * a0;
        const double* yi = st.y + sl * D + 3 * a0;
        double part = 0.0;
#pragma unroll
        for (int k = 0; k < WARP_KA; ++k) {
            const int la = lane + 32 * k;
            if (la < n) {
#pragma unroll
                for (int c = 0; c < 3; ++c) part += yi[3 * la + c] * q[3 * k + c];
            }
        }
        const double b = st.rho[sl * ns + m] * warp_sum_d(part);
        const double ab = alpha[i] - b;
#pragma unroll
        for (int k = 0; k < WARP_KA; ++k) {
            const int la = lane + 32 * k;
            if (la < n) {
#pragma unroll
                for (int c = 0; c < 3; ++c) q[3 * k + c] += si[3 * la + c] * ab;
            }
        }
    }
    // 3. p = -z, zero for a converged system; longest per-atom step (determine_step, :865-884)
    const bool conv = st.converged[m] != 0;
    double longest2 = 0.0;
#pragma unroll
    for (int k = 0; k < WARP_KA; ++k) {
#pragma unroll
        for (int c = 0; c < 3; ++c) q[3 * k + c] = conv ? 0.0 : -q[3 * k + c];
        if (lane + 32 * k < n) {
            const double x = q[3 * k], y = q[3 * k + 1], z = q[3 * k + 2];
            longest2 = fmax(longest2, dot3_rn(x, y, z, x, y, z));
        }
    }
    const double longest = sqrt(warp_max_d(longest2));
    const bool cap = longest >= st.maxstep;
    const double scale = cap ? st.maxstep / longest : 1.0;
    // 4. positions
#pragma unroll
    for (int k = 0; k < WARP_KA; ++k) {
        const int la = lane + 32 * k;
        if (la < n) {
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const int64_t e = 3 * (a0 + la) + c;
                const double p = cap ? q[3 * k + c] * scale : q[3 * k + c];
                const double r = st.r[e];
                const double rn = r + p * st.damping;
                st.p[e] = p;
                st.r0[e] = r;
                st.f0[e] = optimizer_force(st.fixed && st.fixed[a0 + la], forces, st.force_conversion, a0 + la, c);
                st.r[e] = rn;
                st.model_positions[e] = (float)(rn / st.position_conversion);
            }
        }
    }
}

// ---- cluster per system --------------------------------------------------------------------------------------------
template <bool IS_MAX>
__device__ __forceinline__ double cluster_reduce(double v, double* red, double* part, int& phase,
                                                 cg::cluster_group& cl) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = IS_MAX ? warp_max_d(v) : warp_sum_d(v);
    if (lane == 0) red[wid] = v;
    __syncthreads();
    if (wid == 0) {
        double x = lane < RELAX_CL_T / 32 ? red[lane] : 0.0;
        x = IS_MAX ? warp_max_d(x) : warp_sum_d(x);
        if (lane == 0) part[phase] = x;
    }
    cl.sync();
    double tot = 0.0;
#pragma unroll
    for (int r = 0; r < RELAX_CL_CTAS; ++r) {
        const double x = *cl.map_shared_rank(part + phase, r);
        tot = IS_MAX ? fmax(tot, x) : tot + x;
    }
    phase ^= 1;          // the next reduction writes the other slot while slower CTAs may still read this one
    return tot;
}

__global__ void __cluster_dims__(RELAX_CL_CTAS, 1, 1) __launch_bounds__(RELAX_CL_T)
    k_lbfgs_cluster(spk_lbfgs_t st, const float* __restrict__ forces) {
    extern __shared__ double alpha[];                     // [memory], the same values in every CTA of the cluster
    __shared__ double red[RELAX_CL_T / 32];
    __shared__ double part[2];
    SPK_PDL_ENTER();
    cg::cluster_group cl = cg::this_cluster();
    int phase = 0;
    const int64_t it = st.counter[0];
    if (blockIdx.x == 0 && threadIdx.x == 0) st.counter[1] = it + 1;
    const int64_t m = st.order[st.n_warp + blockIdx.x / RELAX_CL_CTAS];
    const int64_t a0 = st.sys_ptr[m];
    const int64_t n = st.sys_ptr[m + 1] - a0;
    const int64_t D = 3 * st.n_atoms;
    const int64_t M = st.memory;
    const int64_t ns = st.n_sys;
    const int64_t G = (int64_t)RELAX_CL_CTAS * RELAX_CL_T;
    const int64_t g = (int64_t)cl.block_rank() * RELAX_CL_T + threadIdx.x;
    double* q = st.p;                                     // the direction, element e owned by the thread of its atom

    double ys = 0.0;
    for (int64_t la = g; la < n; la += G) {
        for (int c = 0; c < 3; ++c) {
            const int64_t e = 3 * (a0 + la) + c;
            const double f = optimizer_force(st.fixed && st.fixed[a0 + la], forces, st.force_conversion, a0 + la, c);
            if (it > 0) {
                const int64_t sl = (it - 1) % M;
                const double s = st.r[e] - st.r0[e];
                const double y = st.f0[e] - f;
                st.s[sl * D + e] = s;
                st.y[sl * D + e] = y;
                ys += y * s;
            }
            q[e] = -f;
        }
    }
    if (it > 0) {
        ys = cluster_reduce<false>(ys, red, part, phase, cl);
        if (g == 0) st.rho[((it - 1) % M) * ns + m] = ys > 1e-8 ? 1.0 / ys : 1.0;
    }
    // rho of the new entry is read below by every CTA: recompute it locally instead of waiting for the store
    const int64_t L = it < M ? it : M;
    auto rho_of = [&](int64_t sl) {
        if (it > 0 && sl == (it - 1) % M) return ys > 1e-8 ? 1.0 / ys : 1.0;
        return st.rho[sl * ns + m];
    };
    for (int64_t i = L - 1; i >= 0; --i) {
        const int64_t sl = (it - L + i) % M;
        const double* si = st.s + sl * D;
        const double* yi = st.y + sl * D;
        double pt = 0.0;
        for (int64_t la = g; la < n; la += G)
            for (int c = 0; c < 3; ++c) {
                const int64_t e = 3 * (a0 + la) + c;
                pt += si[e] * q[e];
            }
        const double a = rho_of(sl) * cluster_reduce<false>(pt, red, part, phase, cl);
        if (threadIdx.x == 0) alpha[i] = a;
        for (int64_t la = g; la < n; la += G)
            for (int c = 0; c < 3; ++c) {
                const int64_t e = 3 * (a0 + la) + c;
                q[e] -= a * yi[e];
            }
    }
    for (int64_t la = g; la < n; la += G)
        for (int c = 0; c < 3; ++c) q[3 * (a0 + la) + c] *= st.h0;
    for (int64_t i = 0; i < L; ++i) {
        const int64_t sl = (it - L + i) % M;
        const double* si = st.s + sl * D;
        const double* yi = st.y + sl * D;
        double pt = 0.0;
        for (int64_t la = g; la < n; la += G)
            for (int c = 0; c < 3; ++c) {
                const int64_t e = 3 * (a0 + la) + c;
                pt += yi[e] * q[e];
            }
        const double b = rho_of(sl) * cluster_reduce<false>(pt, red, part, phase, cl);
        const double ab = alpha[i] - b;                    // alpha[i] was stored before an earlier cluster barrier
        for (int64_t la = g; la < n; la += G)
            for (int c = 0; c < 3; ++c) {
                const int64_t e = 3 * (a0 + la) + c;
                q[e] += si[e] * ab;
            }
    }
    const bool conv = st.converged[m] != 0;
    double longest2 = 0.0;
    for (int64_t la = g; la < n; la += G) {
        const int64_t e = 3 * (a0 + la);
        double* v = q + e;
        for (int c = 0; c < 3; ++c) v[c] = conv ? 0.0 : -v[c];
        longest2 = fmax(longest2, dot3_rn(v[0], v[1], v[2], v[0], v[1], v[2]));
    }
    const double longest = sqrt(cluster_reduce<true>(longest2, red, part, phase, cl));
    const bool cap = longest >= st.maxstep;
    const double scale = cap ? st.maxstep / longest : 1.0;
    for (int64_t la = g; la < n; la += G)
        for (int c = 0; c < 3; ++c) {
            const int64_t e = 3 * (a0 + la) + c;
            const double p = cap ? q[e] * scale : q[e];
            const double r = st.r[e];
            const double rn = r + p * st.damping;
            st.p[e] = p;
            st.r0[e] = r;
            st.f0[e] = optimizer_force(st.fixed && st.fixed[a0 + la], forces, st.force_conversion, a0 + la, c);
            st.r[e] = rn;
            st.model_positions[e] = (float)(rn / st.position_conversion);
        }
    cl.sync();            // no CTA may leave while another still reads its shared memory
}

// ---- convergence (BatchwiseOptimizer.converged, :560-567, and the per-system mask of step, :773-781) -------------
__global__ void __launch_bounds__(CONV_WARPS * 32) k_relax_converged(spk_lbfgs_t st, const float* __restrict__ forces) {
    SPK_PDL_ENTER();
    const int lane = threadIdx.x & 31;
    const int64_t m = (int64_t)blockIdx.x * CONV_WARPS + (threadIdx.x >> 5);
    if (m >= st.n_sys) return;
    const int64_t a0 = st.sys_ptr[m], a1 = st.sys_ptr[m + 1];
    double mx = 0.0;
    for (int64_t a = a0 + lane; a < a1; a += 32) {
        const double x = optimizer_force(st.fixed && st.fixed[a], forces, st.force_conversion, a, 0);
        const double y = optimizer_force(st.fixed && st.fixed[a], forces, st.force_conversion, a, 1);
        const double z = optimizer_force(st.fixed && st.fixed[a], forces, st.force_conversion, a, 2);
        mx = fmax(mx, dot3_rn(x, y, z, x, y, z));
    }
    mx = warp_max_d(mx);
    if (lane == 0) record_convergence(st, m, mx);
}

SpkSmemOnce g_warp_smem, g_cluster_smem;

bool lbfgs_valid(const spk_lbfgs_t* st) {
    return st && st->r && st->r0 && st->f0 && st->s && st->y && st->rho && st->p && st->counter && st->fmax &&
           st->fmax_sys && st->converged && st->steps && st->n_unconverged && st->model_positions && st->sys_ptr &&
           st->order && st->n_atoms >= 0 && st->n_sys >= 1 && st->n_warp >= 0 && st->n_warp <= st->n_sys &&
           st->memory >= 1 && st->position_conversion != 0.0;
}

}  // namespace

extern "C" int spk_relax_step(const spk_lbfgs_t* st, const float* forces, spk_stream_t stream) {
    if (!lbfgs_valid(st) || !forces) return SPK_ERR_ARG;
    if (st->memory > SPK_RELAX_MAX_MEMORY) return SPK_ERR_UNSUPPORTED;
    const cudaStream_t s = spk_st(stream);
    const int64_t n_cluster = st->n_sys - st->n_warp;
    if (st->n_warp > 0) {
        const int smem = (int)(WARP_CTA_WARPS * st->memory * sizeof(double));
        // the attribute is set once per device, so it covers the largest history the library accepts
        if (g_warp_smem.set(k_lbfgs_warp, (int)(WARP_CTA_WARPS * SPK_RELAX_MAX_MEMORY * sizeof(double))) != cudaSuccess)
            return SPK_ERR_UNSUPPORTED;
        spk_launch(k_lbfgs_warp, (unsigned)spk_cdiv(st->n_warp, WARP_CTA_WARPS), WARP_CTA_WARPS * 32, smem, s, *st,
                   forces);
        SPK_LAUNCH_CHECK();
    }
    if (n_cluster > 0) {
        const int smem = (int)(st->memory * sizeof(double));
        if (g_cluster_smem.set(k_lbfgs_cluster, (int)(SPK_RELAX_MAX_MEMORY * sizeof(double))) != cudaSuccess)
            return SPK_ERR_UNSUPPORTED;
        spk_launch(k_lbfgs_cluster, (unsigned)(n_cluster * RELAX_CL_CTAS), RELAX_CL_T, smem, s, *st, forces);
        SPK_LAUNCH_CHECK();
    }
    return SPK_OK;
}

extern "C" int spk_relax_converged(const spk_lbfgs_t* st, const float* forces, spk_stream_t stream) {
    if (!lbfgs_valid(st) || !forces) return SPK_ERR_ARG;
    const cudaStream_t s = spk_st(stream);
    spk_launch(k_relax_converged, (unsigned)spk_cdiv(st->n_sys, CONV_WARPS), CONV_WARPS * 32, 0, s, *st, forces);
    SPK_LAUNCH_CHECK();
    spk_launch(k_count_unconverged<spk_lbfgs_t>, 1, 256, 0, s, *st);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

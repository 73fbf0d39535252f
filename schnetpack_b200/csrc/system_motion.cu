// Set-up and steadying of the device MD state (md/system.py:258-315,652-684, md/initial_conditions.py:50-188,
// md/simulation_hooks/basic_hooks.py:55-78): centre-of-mass, translation and rotation removal, position wrapping and the
// initial momenta of the Maxwell-Boltzmann and uniform initializers.  Every entry point only enqueues work, so the hooks
// can run inside a captured step.
//
// Motion removal is three launches.  k_motion_partials sums, per (system, CTA) pair, the fp64 terms of every atom taken
// relative to its system's first atom x_r (y = x - x_r, so a system far from the origin loses no digits): m, m y, p and,
// for the rotation, y, the upper triangle of m y y^T and y x p.  k_motion_solve adds a system's partials in CTA order
// (seg_finish_block), forms the centre of mass c, the mean momentum and, with the parallel-axis identities, the inertia
// tensor and the angular momentum about the origin of the shifted positions; its first thread solves I w = L by the
// eigenvalues of I (sym3_eig), dropping those at or below SPK_MOTION_PINV_RTOL x the largest, so a single atom or a
// linear molecule gets the pseudo-inverse.  k_motion_apply writes x - c and p - p_mean - m (w x (x - c)).  No atomics:
// the results are bitwise the same on every call, for any mix of system sizes.
//
// The hook kernels read the device step counter step[0] and return at once unless step[0] % every == 0, so one captured
// step serves every step of the run.
#include "md_common.cuh"

namespace {

constexpr int MOT_T = 128;   // atoms per CTA of the partial pass
constexpr int MOT_COEF = 9;  // per-system coefficients: c[3], p_mean[3], w[3]

template <bool ROT>
struct MotionTerms {
    static constexpr int NV = ROT ? 19 : 7;   // m, m y[3], p[3] (+ y[3], m yy^T[6], y x p[3])
};

static inline int64_t mot_blocks(int64_t n_atoms) { return spk_cdiv(n_atoms, MOT_T); }

__device__ __forceinline__ bool gated_off(const int64_t* step, int64_t every) {
    return step != nullptr && (*step) % every != 0;
}

template <bool ROT>
__global__ void __launch_bounds__(MOT_T) k_motion_partials(const float* __restrict__ x, const float* __restrict__ p,
                                                           const float* __restrict__ m, const int64_t* __restrict__ idx_m,
                                                           const int32_t* __restrict__ sys_ptr, int64_t n_atoms,
                                                           const int64_t* __restrict__ step, int64_t every,
                                                           double* __restrict__ sys_part, double* __restrict__ head) {
    constexpr int NV = MotionTerms<ROT>::NV;
    SPK_PDL_ENTER();
    if (gated_off(step, every)) return;
    const int64_t a = (int64_t)blockIdx.x * MOT_T + threadIdx.x;
    double v[NV];
#pragma unroll
    for (int c = 0; c < NV; ++c) v[c] = 0.0;
    int64_t s = 0, first = 0, end = 0;
    if (a < n_atoms) {
        s = idx_m[a];
        first = sys_ptr[s];
        end = sys_ptr[s + 1];
        const double y0 = (double)x[3 * a] - (double)x[3 * first];
        const double y1 = (double)x[3 * a + 1] - (double)x[3 * first + 1];
        const double y2 = (double)x[3 * a + 2] - (double)x[3 * first + 2];
        const double p0 = p[3 * a], p1 = p[3 * a + 1], p2 = p[3 * a + 2];
        const double ma = m[a];
        v[0] = ma;
        v[1] = ma * y0; v[2] = ma * y1; v[3] = ma * y2;
        v[4] = p0; v[5] = p1; v[6] = p2;
        if constexpr (ROT) {
            v[7] = y0; v[8] = y1; v[9] = y2;
            v[10] = ma * y0 * y0; v[11] = ma * y1 * y1; v[12] = ma * y2 * y2;
            v[13] = ma * y0 * y1; v[14] = ma * y0 * y2; v[15] = ma * y1 * y2;
            v[16] = y1 * p2 - y2 * p1; v[17] = y2 * p0 - y0 * p2; v[18] = y0 * p1 - y1 * p0;
        }
    }
    seg_partials<MOT_T, NV>(v, n_atoms, s, first, end, sys_part, head);
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* out) {
    out[0] = a[1] * b[2] - a[2] * b[1];
    out[1] = a[2] * b[0] - a[0] * b[2];
    out[2] = a[0] * b[1] - a[1] * b[0];
}

// one CTA per system: the ordered totals, then thread 0 forms c, p_mean and w (system.py:258-315)
template <bool ROT>
__global__ void __launch_bounds__(SEG_FIN_T) k_motion_solve(const float* __restrict__ x, const int32_t* __restrict__ sys_ptr,
                                                            int flags, const int64_t* __restrict__ step, int64_t every,
                                                            const double* __restrict__ sys_part,
                                                            const double* __restrict__ head, double* __restrict__ coef) {
    constexpr int NV = MotionTerms<ROT>::NV;
    __shared__ double red[NV][SEG_FIN_T];
    SPK_PDL_ENTER();
    if (gated_off(step, every)) return;
    const int64_t s = blockIdx.x;
    seg_finish_block<MOT_T, NV>(sys_ptr, nullptr, sys_part, head, s, red);
    if (threadIdx.x != 0) return;
    double* out = coef + s * MOT_COEF;
    const int64_t a0 = sys_ptr[s], n = sys_ptr[s + 1] - a0;
    double S[NV];
#pragma unroll
    for (int c = 0; c < NV; ++c) S[c] = red[c][0];
    double c[3] = {0.0, 0.0, 0.0}, q[3] = {0.0, 0.0, 0.0}, w[3] = {0.0, 0.0, 0.0}, xr[3] = {0.0, 0.0, 0.0};
    if (n > 0) {
        for (int k = 0; k < 3; ++k) xr[k] = x[3 * a0 + k];
        const double M = S[0];
        if ((flags & SPK_MOTION_CENTER_OF_MASS) && M > 0.0)              // :258-276, x -= sum m x / sum m
            for (int k = 0; k < 3; ++k) c[k] = xr[k] + S[1 + k] / M;
        if (flags & SPK_MOTION_TRANSLATION)                               // :278-283, unweighted mean of p
            for (int k = 0; k < 3; ++k) q[k] = S[4 + k] / (double)n;
        if constexpr (ROT) {
            // positions x' = y + d with d = x_r - c, momenta p' = p - q; about the origin (:285-315):
            // A = sum m x' x'^T = S_myy + d S_my^T + S_my d^T + M d d^T, I = tr(A) 1 - A,
            // L = sum x' x p' = S_yxp + d x S_p - S_y x q - n d x q
            double d[3], A[3][3];
            for (int k = 0; k < 3; ++k) d[k] = xr[k] - c[k];
            const double syy[3][3] = {{S[10], S[13], S[14]}, {S[13], S[11], S[15]}, {S[14], S[15], S[12]}};
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) A[i][j] = syy[i][j] + d[i] * S[1 + j] + S[1 + i] * d[j] + M * d[i] * d[j];
            const double tr = A[0][0] + A[1][1] + A[2][2];
            double I[9];
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) I[i * 3 + j] = (i == j ? tr : 0.0) - A[i][j];
            double L[3], t1[3], t2[3], t3[3];
            cross3(d, S + 4, t1);
            cross3(S + 7, q, t2);
            cross3(d, q, t3);
            for (int k = 0; k < 3; ++k) L[k] = S[16 + k] + t1[k] - t2[k] - (double)n * t3[k];
            double lam[3], V[3][3];
            sym3_eig(I, lam, V);
            const double lmax = fmax(lam[0], fmax(lam[1], lam[2]));
            for (int e = 0; e < 3; ++e) {
                if (!(lam[e] > SPK_MOTION_PINV_RTOL * lmax)) continue;     // singular direction: no rotation about it
                const double proj = (V[0][e] * L[0] + V[1][e] * L[1] + V[2][e] * L[2]) / lam[e];
                for (int k = 0; k < 3; ++k) w[k] += proj * V[k][e];
            }
        }
    }
    for (int k = 0; k < 3; ++k) {
        out[k] = c[k];
        out[3 + k] = q[k];
        out[6 + k] = w[k];
    }
}

// one thread per atom: x -= c (and the model-unit copy), p -= p_mean + m (w x (x - c))
__global__ void k_motion_apply(float* __restrict__ x, float* __restrict__ mx, float* __restrict__ p,
                               const float* __restrict__ m, const int64_t* __restrict__ idx_m, int64_t n_atoms, int flags,
                               float p_conv, const int64_t* __restrict__ step, int64_t every,
                               const double* __restrict__ coef) {
    SPK_PDL_ENTER();
    if (gated_off(step, every)) return;
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const double* cf = coef + idx_m[a] * MOT_COEF;
    double xs[3];
    for (int k = 0; k < 3; ++k) xs[k] = (double)x[3 * a + k] - cf[k];
    if (flags & SPK_MOTION_CENTER_OF_MASS) {
        for (int k = 0; k < 3; ++k) {
            const float xf = (float)xs[k];
            x[3 * a + k] = xf;
            if (mx) mx[3 * a + k] = xf * p_conv;
        }
    }
    if (flags & (SPK_MOTION_TRANSLATION | SPK_MOTION_ROTATION)) {
        double r[3];
        cross3(cf + 6, xs, r);
        const double ma = m[a];
        for (int k = 0; k < 3; ++k) p[3 * a + k] = (float)((double)p[3 * a + k] - cf[3 + k] - ma * r[k]);
    }
}

// system.py:652-684 for the P beads of one atom: the lattice translation n = floor(f_c + eps) of the centroid's
// fractional coordinates f_c = x_c C^-1 (periodic axes only) moves every bead, x_k -= n C.  P = 1 is the reference's
// ((f + eps) mod 1) - eps.  The cell of atom a is that of its bead-0 system idx_m[a].
__global__ void k_wrap_positions(float* __restrict__ x, float* __restrict__ mx, const int64_t* __restrict__ idx_m,
                                 int64_t n_atoms, int n_beads, const double* __restrict__ cell, int64_t cell_stride,
                                 const uint8_t* __restrict__ pbc, int64_t pbc_stride, double eps, float p_conv,
                                 const int64_t* __restrict__ step, int64_t every) {
    SPK_PDL_ENTER();
    if (gated_off(step, every)) return;
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const int64_t s = idx_m[a];
    const double* C = cell + s * cell_stride;
    const uint8_t* per = pbc + s * pbc_stride;
    double xc[3] = {0.0, 0.0, 0.0};
    for (int k = 0; k < n_beads; ++k)
        for (int j = 0; j < 3; ++j) xc[j] += (double)x[3 * (k * n_atoms + a) + j];
    for (int j = 0; j < 3; ++j) xc[j] /= (double)n_beads;
    // f = x C^-1 = x adj(C) / det(C), adj(C)[i][j] = cofactor(C)[j][i]
    const double det = det3(C);
    const double inv[3][3] = {
        {(C[4] * C[8] - C[5] * C[7]) / det, (C[2] * C[7] - C[1] * C[8]) / det, (C[1] * C[5] - C[2] * C[4]) / det},
        {(C[5] * C[6] - C[3] * C[8]) / det, (C[0] * C[8] - C[2] * C[6]) / det, (C[2] * C[3] - C[0] * C[5]) / det},
        {(C[3] * C[7] - C[4] * C[6]) / det, (C[1] * C[6] - C[0] * C[7]) / det, (C[0] * C[4] - C[1] * C[3]) / det}};
    double shift[3] = {0.0, 0.0, 0.0};
    bool moved = false;
    for (int j = 0; j < 3; ++j) {
        if (!per[j]) continue;
        const double f = xc[0] * inv[0][j] + xc[1] * inv[1][j] + xc[2] * inv[2][j];
        const double nj = floor(f + eps);
        if (nj != 0.0) {
            moved = true;
            for (int i = 0; i < 3; ++i) shift[i] += nj * C[j * 3 + i];
        }
    }
    if (!moved) return;
    for (int k = 0; k < n_beads; ++k) {
        const int64_t r = 3 * (k * n_atoms + a);
        for (int j = 0; j < 3; ++j) {
            const float xf = (float)((double)x[r + j] - shift[j]);
            x[r + j] = xf;
            if (mx) mx[r + j] = xf * p_conv;
        }
    }
}

// initial_conditions.py:119-135,169-188: p = w xi with w = m (uniform) or sqrt(m kB T_s) (Maxwell-Boltzmann); xi from
// Philox4x32-10 keyed by seed with the counter (atom, SPK_MOTION_DRAW_APPLICATION), normals 0..2 for x, y, z as in
// spk_md_langevin
__global__ void k_initial_momenta(float* __restrict__ p, const float* __restrict__ m, const int64_t* __restrict__ idx_m,
                                  int64_t n_atoms, int uniform, double kB, const double* __restrict__ temperature,
                                  uint64_t seed) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const uint4 r = philox_draw(seed, SPK_MOTION_DRAW_APPLICATION, a);
    const double2 z01 = box_muller(r.x, r.y), z23 = box_muller(r.z, r.w);
    const double ma = m[a];
    const double w = uniform ? ma : sqrt(ma * kB * temperature[idx_m[a]]);
    p[3 * a + 0] = (float)(w * z01.x);
    p[3 * a + 1] = (float)(w * z01.y);
    p[3 * a + 2] = (float)(w * z23.x);
}

// UniformInit's exact rescale: p *= sqrt(T_target / T) per system, a system with T = 0 left as it is
__global__ void k_rescale_temperature(float* __restrict__ p, const int64_t* __restrict__ idx_m, int64_t n,
                                      const double* __restrict__ target, const double* __restrict__ current) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int64_t s = idx_m[i / 3];
    const double t = current[s];
    if (t > 0.0) p[i] = (float)(sqrt(target[s] / t) * (double)p[i]);
}

__global__ void k_step_advance(int64_t* __restrict__ step) {
    SPK_PDL_ENTER();
    if (threadIdx.x == 0) step[0] += 1;
}

static int check_layout(const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys) {
    if (n_atoms < 0 || n_sys <= 0 || n_atoms >= (1ll << 31) / 3) return SPK_ERR_ARG;
    if (!sys_ptr || (n_atoms > 0 && !idx_m)) return SPK_ERR_ARG;
    return SPK_OK;
}

}  // namespace

extern "C" size_t spk_md_motion_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? mot_blocks(n_atoms) : 0;
    const int64_t ns = n_sys > 0 ? n_sys : 0;
    const size_t own = sizeof(double) * (size_t)((MotionTerms<true>::NV + MOT_COEF) * ns + MotionTerms<true>::NV * nb + 1);
    const size_t init = sizeof(double) * (size_t)(2 * ns) + spk_md_thermostat_workspace_bytes(n_atoms, n_sys);
    return own > init ? own : init;
}

extern "C" int spk_md_remove_motion(float* positions, float* model_positions, float* momenta, const float* masses,
                                    const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys,
                                    int flags, float position_conversion, const int64_t* step, int64_t every,
                                    void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    int rc = check_layout(idx_m, sys_ptr, n_atoms, n_sys);
    if (rc != SPK_OK) return rc;
    if (flags & ~(SPK_MOTION_CENTER_OF_MASS | SPK_MOTION_TRANSLATION | SPK_MOTION_ROTATION) || every < 1) return SPK_ERR_ARG;
    if (!workspace || workspace_bytes < spk_md_motion_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    if (flags == 0 || n_atoms == 0) return SPK_OK;
    if (!positions || !momenta || !masses) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    const bool rot = flags & SPK_MOTION_ROTATION;
    const int nv = rot ? MotionTerms<true>::NV : MotionTerms<false>::NV;
    double* coef = reinterpret_cast<double*>(workspace);
    double* sys_part = coef + MOT_COEF * n_sys;
    double* head = sys_part + (int64_t)nv * n_sys;
    const unsigned nb = (unsigned)mot_blocks(n_atoms);
    if (rot) {
        spk_launch(k_motion_partials<true>, nb, MOT_T, 0, st, positions, momenta, masses, idx_m, sys_ptr, n_atoms, step,
                   every, sys_part, head);
        spk_launch(k_motion_solve<true>, (unsigned)n_sys, SEG_FIN_T, 0, st, positions, sys_ptr, flags, step, every,
                   sys_part, head, coef);
    } else {
        spk_launch(k_motion_partials<false>, nb, MOT_T, 0, st, positions, momenta, masses, idx_m, sys_ptr, n_atoms, step,
                   every, sys_part, head);
        spk_launch(k_motion_solve<false>, (unsigned)n_sys, SEG_FIN_T, 0, st, positions, sys_ptr, flags, step, every,
                   sys_part, head, coef);
    }
    spk_launch(k_motion_apply, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, positions, model_positions, momenta, masses,
               idx_m, n_atoms, flags, position_conversion, step, every, coef);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_wrap_positions(float* positions, float* model_positions, const int64_t* idx_m, int64_t n_atoms,
                                     int32_t n_beads, const double* cell, int64_t cell_stride, const uint8_t* pbc,
                                     int64_t pbc_stride, double eps, float position_conversion, const int64_t* step,
                                     int64_t every, spk_stream_t stream) {
    if (n_atoms < 0 || n_beads < 1 || n_atoms * n_beads >= (1ll << 31) / 3 || every < 1) return SPK_ERR_ARG;
    if ((cell_stride != 0 && cell_stride != 9) || (pbc_stride != 0 && pbc_stride != 3)) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!positions || !idx_m || !cell || !pbc) return SPK_ERR_ARG;
    spk_launch(k_wrap_positions, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, spk_st(stream), positions, model_positions,
               idx_m, n_atoms, (int)n_beads, cell, cell_stride, pbc, pbc_stride, eps, position_conversion, step, every);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_initial_momenta(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                                      int64_t n_atoms, int64_t n_sys, int uniform, double kB, const double* temperature,
                                      uint64_t seed, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    int rc = check_layout(idx_m, sys_ptr, n_atoms, n_sys);
    if (rc != SPK_OK) return rc;
    if (!(kB > 0.0) || !temperature) return SPK_ERR_ARG;
    if (!workspace || workspace_bytes < spk_md_motion_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!momenta || !masses) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    spk_launch(k_initial_momenta, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, momenta, masses, idx_m, n_atoms, uniform,
               kB, temperature, seed);
    SPK_LAUNCH_CHECK();
    if (!uniform) return SPK_OK;
    // the fixed-order kinetic sum of the thermostats, then the rescale
    double* current = reinterpret_cast<double*>(workspace);
    double* ke = current + n_sys;
    void* ws = ke + n_sys;
    const size_t ws_bytes = workspace_bytes - sizeof(double) * (size_t)(2 * n_sys);
    rc = spk_md_kinetic_energy(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, kB, ke, current, ws, ws_bytes, stream);
    if (rc != SPK_OK) return rc;
    spk_launch(k_rescale_temperature, (unsigned)spk_cdiv(3 * n_atoms, 256), 256, 0, st, momenta, idx_m, 3 * n_atoms,
               temperature, current);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_step_advance(int64_t* step, spk_stream_t stream) {
    if (!step) return SPK_ERR_ARG;
    spk_launch(k_step_advance, 1, 32, 0, spk_st(stream), step);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

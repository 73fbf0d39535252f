// Statistics of a model ensemble (md/calculators/ensemble_calculator.py:38-59, interfaces/batchwise_optimization.py:
// 36-72, interfaces/ase_interface.py:340-432): the K members' fp32 outputs sit in stacked slots [K, ...], and these
// kernels reduce them over k in fp64.
//
// Every mean and spread takes two passes over k in ascending order: the mean first, then the sum of squared deviations
// from it.  The one-pass form sum x^2 - (sum x)^2 / K cancels catastrophically when the spread is small next to the mean
// (energies of 1e4 with a spread of 1e-3 lose every digit of the variance in fp32 and most of them in fp64).  The per-atom
// force terms are summed per system by the partial pass of segscan.cuh (seg_partials over EF_T consecutive atoms, then
// k_seg_finish), so no sum uses atomics and every result is bitwise reproducible.
#include "common.cuh"
#include "segscan.cuh"

namespace {

constexpr int EM_T = 256;   // elements per CTA of the element-wise moments
constexpr int EF_T = 128;   // atoms per CTA of the force statistics and of their partial pass
constexpr int EU_T = 128;   // systems per CTA of the uncertainty
constexpr int EF_NV = 2;    // per-atom terms summed per system: ||std_0(F_i)||, ||std_0(F_i)|| / (||mean(F_i)|| + 1e-8)
constexpr double REL_EPS = 1e-8;   // ase_interface.py:402,414,427

// mean and sum of squared deviations of x[k * stride], k = 0..K-1, each scaled by `scale` first
__device__ __forceinline__ void two_pass(const float* __restrict__ x, int64_t K, int64_t stride, double scale,
                                         double& mean, double& ss) {
    double s = 0.0;
    for (int64_t k = 0; k < K; ++k) s += (double)x[k * stride] * scale;
    mean = s / (double)K;
    ss = 0.0;
    for (int64_t k = 0; k < K; ++k) {
        const double d = (double)x[k * stride] * scale - mean;
        ss += d * d;
    }
}

__global__ void __launch_bounds__(EM_T) k_ensemble_moments(const float* __restrict__ x, int64_t K, int64_t n, int ddof,
                                                           double mean_scale, double spread_scale,
                                                           float* __restrict__ mean, float* __restrict__ var,
                                                           float* __restrict__ std) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)EM_T + threadIdx.x;
    if (i >= n) return;
    double mu, ss;
    two_pass(x + i, K, n, 1.0, mu, ss);
    const double v = ss / (double)(K - ddof);
    if (mean) mean[i] = (float)(mu * mean_scale);
    if (var) var[i] = (float)(v * spread_scale);
    if (std) std[i] = (float)(sqrt(v) * spread_scale);
}

// one thread per atom: mean and unbiased variance of each component over the K slots, the per-atom uncertainty terms
// (of the values times spread_scale, ddof 0 as np.std) and their per-system partials
__global__ void __launch_bounds__(EF_T) k_ensemble_forces(const float* __restrict__ f, int64_t K, int64_t n_atoms,
                                                          const int64_t* __restrict__ idx_m,
                                                          const int32_t* __restrict__ sys_ptr, double mean_scale,
                                                          double spread_scale, float* __restrict__ mean,
                                                          float* __restrict__ var, double* __restrict__ sys_part,
                                                          double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * EF_T + threadIdx.x;
    double v[EF_NV] = {0.0, 0.0};
    int64_t m = 0, first = 0, end = 0;
    if (a < n_atoms) {
        double sd2 = 0.0, mu2 = 0.0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            double mu, ss;
            two_pass(f + 3 * a + c, K, 3 * n_atoms, 1.0, mu, ss);
            if (mean) mean[3 * a + c] = (float)(mu * mean_scale);
            if (var) var[3 * a + c] = (float)(ss / (double)(K - 1) * spread_scale);
            const double mus = mu * spread_scale;
            sd2 += ss / (double)K * (spread_scale * spread_scale);
            mu2 += mus * mus;
        }
        const double sd = sqrt(sd2);
        v[0] = sd;
        v[1] = sd / (sqrt(mu2) + REL_EPS);
        if (sys_part) {
            m = idx_m[a];
            first = sys_ptr[m];
            end = sys_ptr[m + 1];
        }
    }
    if (sys_part) seg_partials<EF_T, EF_NV>(v, n_atoms, m, first, end, sys_part, head);
}

// ||std_0|| row norms of a [K, 3, 3] stack (stride between slots: `stride` floats), averaged over the rows; relative:
// each row norm over (||mean row|| + 1e-8) first (ase_interface.py:381-388,419-429).  Out of line: inlined next to the
// energy term, the calls of the fp64 division slow path make ptxas spill.
__device__ __noinline__ double stress_term(const float* __restrict__ s, int64_t K, int64_t stride, double scale,
                                              int relative) {
    double acc = 0.0;
    for (int r = 0; r < 3; ++r) {
        double sd2 = 0.0, mu2 = 0.0;
        for (int c = 0; c < 3; ++c) {
            double mu, ss;
            two_pass(s + 3 * r + c, K, stride, scale, mu, ss);
            sd2 += ss / (double)K;
            mu2 += mu * mu;
        }
        const double t = sqrt(sd2);
        acc += relative ? t / (sqrt(mu2) + REL_EPS) : t;
    }
    return acc / 3.0;
}

// one thread per system: the weighted sum of the energy, force and stress terms (ase_interface.py:365-432)
__global__ void __launch_bounds__(EU_T) k_ensemble_uncertainty(const float* __restrict__ energy, double energy_scale,
                                                               const double* __restrict__ force_sums,
                                                               const int32_t* __restrict__ sys_ptr,
                                                               const float* __restrict__ stress, double stress_scale,
                                                               int64_t K, int64_t n_sys, int relative, double w_e,
                                                               double w_f, double w_s, double* __restrict__ out,
                                                               float* __restrict__ out_f32) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)EU_T + threadIdx.x;
    if (s >= n_sys) return;
    double u = 0.0;
    if (w_e > 0.0) {
        double mu, ss;
        two_pass(energy + s, K, n_sys, energy_scale, mu, ss);
        const double sd = sqrt(ss / (double)K);
        u += w_e * (relative ? sd / (fabs(mu) + REL_EPS) : sd);
    }
    if (w_f > 0.0) {
        // mean over the system's atoms; a system without atoms contributes 0 (np.mean of nothing would be NaN)
        const int64_t n = sys_ptr[s + 1] - sys_ptr[s];
        if (n > 0) u += w_f * (force_sums[s * EF_NV + (relative ? 1 : 0)] / (double)n);
    }
    if (w_s > 0.0) u += w_s * stress_term(stress + 9 * s, K, 9 * n_sys, stress_scale, relative);
    if (out) out[s] = u;
    if (out_f32) out_f32[s] = (float)u;
}

}  // namespace

extern "C" size_t spk_ensemble_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    if (n_atoms < 0 || n_sys < 0) return 0;
    return sizeof(double) * EF_NV * (size_t)(n_sys + spk_cdiv(n_atoms, EF_T));
}

extern "C" int spk_ensemble_moments(const float* x, int64_t K, int64_t n, int ddof, double mean_scale,
                                    double spread_scale, float* mean, float* var, float* std, spk_stream_t stream) {
    if (K < 1 || n < 0 || (ddof != 0 && ddof != 1) || K <= ddof) return SPK_ERR_ARG;
    if (n == 0 || (!mean && !var && !std)) return SPK_OK;
    if (!x) return SPK_ERR_ARG;
    spk_launch(k_ensemble_moments, (unsigned)spk_cdiv(n, EM_T), EM_T, 0, spk_st(stream), x, K, n, ddof, mean_scale,
               spread_scale, mean, var, std);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_ensemble_forces(const float* forces, int64_t K, const int64_t* idx_m, const int32_t* sys_ptr,
                                   int64_t n_atoms, int64_t n_sys, double mean_scale, double spread_scale, float* mean,
                                   float* var, double* sys_terms, void* workspace, size_t workspace_bytes,
                                   spk_stream_t stream) {
    if (K < 2 || n_atoms < 0 || n_atoms >= (1ll << 31) - 1 || n_sys < 0 || n_sys > 0x7fffffff) return SPK_ERR_ARG;
    if (sys_terms) {
        if (n_sys < 1 || !sys_ptr || !workspace || workspace_bytes < spk_ensemble_workspace_bytes(n_atoms, n_sys))
            return SPK_ERR_ARG;
        if (n_atoms > 0 && !idx_m) return SPK_ERR_ARG;
    }
    if (n_atoms > 0 && !forces && (mean || var || sys_terms)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    double* sys_part = sys_terms ? reinterpret_cast<double*>(workspace) : nullptr;
    double* head = sys_terms ? sys_part + EF_NV * n_sys : nullptr;
    if (n_atoms > 0 && (mean || var || sys_terms))
        spk_launch(k_ensemble_forces, (unsigned)spk_cdiv(n_atoms, EF_T), EF_T, 0, st, forces, K, n_atoms, idx_m, sys_ptr,
                   mean_scale, spread_scale, mean, var, sys_part, head);
    if (sys_terms)
        spk_launch(k_seg_finish<EF_T, EF_NV>, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, (const int32_t*)nullptr,
                   (const double*)sys_part, (const double*)head, sys_terms);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_ensemble_uncertainty(const float* energy, double energy_scale, const double* force_sums,
                                        const int32_t* sys_ptr, const float* stress, double stress_scale, int64_t K,
                                        int64_t n_sys, int relative, double energy_weight, double force_weight,
                                        double stress_weight, double* out, float* out_f32, spk_stream_t stream) {
    if (K < 1 || n_sys < 0 || (!out && !out_f32)) return SPK_ERR_ARG;
    if (energy_weight > 0.0 && !energy) return SPK_ERR_ARG;
    if (force_weight > 0.0 && (!force_sums || !sys_ptr)) return SPK_ERR_ARG;
    if (stress_weight > 0.0 && !stress) return SPK_ERR_ARG;
    if (n_sys == 0) return SPK_OK;
    spk_launch(k_ensemble_uncertainty, (unsigned)spk_cdiv(n_sys, EU_T), EU_T, 0, spk_st(stream), energy, energy_scale,
               force_sums, sys_ptr, stress, stress_scale, K, n_sys, relative ? 1 : 0, energy_weight, force_weight,
               stress_weight, out, out_f32);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

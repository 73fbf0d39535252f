// Device code shared by the thermostat (thermostat.cu), barostat (barostat.cu) and ring-polymer (rpmd.cu) kernels of the
// device MD step: the Nose-Hoover chain propagator, the momentum scalings, the Philox4x32-10 generator with its
// application-counter ticket and Box-Muller, the reference's sinh(x)/x series, the cell volume and a 3x3 symmetric Jacobi
// eigensolver.
#pragma once
#include "segscan.cuh"

namespace {

// thermostats.py:398-468 for one chain (barostats.py:408-481 runs the same propagation on the particle and on the cell
// chains); v, f, M point at its chain_length entries and kbt is the chain's kB T (q.kb_temperature, or the bath
// temperature of the chain's system).  Operation order as in the reference.
__device__ double nhc_propagate(double ke, double dof, const spk_nhc_params_t& q, double kbt, double* __restrict__ v,
                                double* __restrict__ f, const double* __restrict__ M) {
    const int L = q.chain_length;
    f[0] = (ke - dof * kbt) / M[0];
    double scaling = 1.0;
    for (int ms = 0; ms < q.multi_step; ++ms) {
        for (int k = 0; k < q.order; ++k) {
            const double h = q.time_step[k];
            v[L - 1] += 0.25 * f[L - 1] * h;
            for (int c = L - 2; c >= 0; --c) {
                const double coeff = exp(-0.125 * h * v[c + 1]);
                v[c] = v[c] * (coeff * coeff) + 0.25 * f[c] * coeff * h;
            }
            scaling *= exp(-0.5 * h * v[0]);
            f[0] = (scaling * scaling * ke - dof * kbt) / M[0];
            for (int c = 0; c < L - 1; ++c) {
                const double coeff = exp(-0.125 * h * v[c + 1]);
                v[c] = v[c] * (coeff * coeff) + 0.25 * f[c] * coeff * h;
                f[c + 1] = (M[c] * (v[c] * v[c]) - kbt) / M[c + 1];
            }
            v[L - 1] += 0.25 * f[L - 1] * h;
        }
    }
    return scaling;
}

__global__ void k_scale_momenta(float* __restrict__ p, const int64_t* __restrict__ idx_m,
                                const double* __restrict__ scale, int64_t n) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    p[i] = (float)(scale[idx_m[i / 3]] * (double)p[i]);
}

// massive NHC: one chain per degree of freedom (thermostats.py:348-354,483-487), one thread per chain.  kbt_sys (nullable)
// holds kB T per system, read through idx_m; without it every chain uses q.kb_temperature.
__global__ void k_nhc_massive(float* __restrict__ p, const float* __restrict__ m, int64_t n_dof,
                              const __grid_constant__ spk_nhc_params_t q, const int64_t* __restrict__ idx_m,
                              const double* __restrict__ kbt_sys, double* __restrict__ chain_v,
                              double* __restrict__ chain_f, const double* __restrict__ chain_m) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_dof) return;
    const double pi = (double)p[i];
    const double ke = pi * pi / (double)m[i / 3];
    const int L = q.chain_length;
    const double kbt = kbt_sys ? kbt_sys[idx_m[i / 3]] : q.kb_temperature;
    const double sc = nhc_propagate(ke, 1.0, q, kbt, chain_v + i * L, chain_f + i * L, chain_m + i * L);
    p[i] = (float)(pi * sc);
}

// ---- Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11) + Box-Muller ---------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k.x += 0x9E3779B9u;
            k.y += 0xBB67AE85u;
        }
        const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
        const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    }
    return c;
}

// counter = (element lo, element hi, application lo, application hi), key = seed
__device__ __forceinline__ uint4 philox_draw(uint64_t seed, uint64_t app, int64_t elem) {
    const uint64_t e = (uint64_t)elem;
    return philox4x32_10(make_uint4((uint32_t)e, (uint32_t)(e >> 32), (uint32_t)app, (uint32_t)(app >> 32)),
                         make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
}

// The application-counter ticket of the noise kernels: counter[0] is the application index every CTA reads at entry,
// counter[1] a ticket, zero between launches.  The CTA that finishes last advances the index, so each replay of a captured
// step draws fresh noise.  Every thread of the CTA calls it after its last use of app.
__device__ __forceinline__ void advance_counter(unsigned long long* counter, unsigned long long app) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(counter + 1, 1ull) == gridDim.x - 1) {
            counter[0] = app + 1;
            counter[1] = 0;
            __threadfence();
        }
    }
}

// u in (0, 1): (x + 1/2) 2^-32; z0 = sqrt(-2 ln u0) cos(2 pi u1), z1 = ... sin(2 pi u1)
__device__ __forceinline__ double2 box_muller(uint32_t x0, uint32_t x1) {
    const double u0 = ((double)x0 + 0.5) * 2.3283064365386963e-10;
    const double u1 = ((double)x1 + 0.5) * 2.3283064365386963e-10;
    const double r = sqrt(-2.0 * log(u0));
    double sn, cs;
    sincospi(2.0 * u1, &sn, &cs);
    return make_double2(r * cs, r * sn);
}

// StableSinhDiv.f of md/utils/thermostat_utils.py:181-201 exactly as written: the series branch is taken for x < eps (not
// |x| < eps), and its polynomial multiplies by x where x^2 is meant, so the "x^4" term is x^3 / 120.  The deviation from
// sinh(x)/x is below |x|^3 / 120, far under every tolerance at realistic dt * v_cell; keeping it makes the device follow the
// reference bit for bit in structure.
__host__ __device__ __forceinline__ double stable_sinh_div(double x) {
    const double e0 = 1.0, e2 = e0 / 6.0, e4 = e2 / 20.0, e6 = e4 / 42.0, e8 = e6 / 72.0, eps = 1e-4;
    const double x2 = x * x;
    if (x < eps) return (((e8 * x2 + e6) * x2 + e4) * x + e2) * x2 + e0;
    return sinh(x) / x;
}

__device__ __forceinline__ double det3(const double* __restrict__ c) {   // system.py:575-580: c0 . (c1 x c2)
    return c[0] * (c[4] * c[8] - c[5] * c[7]) + c[1] * (c[5] * c[6] - c[3] * c[8]) + c[2] * (c[3] * c[7] - c[4] * c[6]);
}

// Eigendecomposition of the symmetric 3x3 matrix whose upper triangle is a[0..8] (row-major; the lower triangle is not
// read, as torch.symeig(upper=True) did): cyclic Jacobi rotations in fp64, one thread, a fixed maximum of sweeps.
// Returns eigenvalues w[k] and eigenvectors as columns of V (V[i][k]).  Any order / sign of the eigenpairs gives the same
// operators Q f(diag w) Q^T, which is all the barostat uses.
__host__ __device__ inline void sym3_eig(const double* __restrict__ a_in, double (&w)[3], double (&V)[3][3]) {
    double a[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            a[i][j] = i <= j ? a_in[i * 3 + j] : a_in[j * 3 + i];
            V[i][j] = i == j ? 1.0 : 0.0;
        }
    const int P[3] = {0, 0, 1}, Q[3] = {1, 2, 2};
    for (int sweep = 0; sweep < 32; ++sweep) {
        const double off = fabs(a[0][1]) + fabs(a[0][2]) + fabs(a[1][2]);
        if (off == 0.0) break;
        for (int r = 0; r < 3; ++r) {
            const int p = P[r], q = Q[r];
            const double apq = a[p][q];
            if (apq == 0.0) continue;
            const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
            const double t = fabs(theta) > 1e150 ? 0.5 / theta
                                                  : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
            const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
            for (int k = 0; k < 3; ++k) {   // A J
                const double akp = a[k][p], akq = a[k][q];
                a[k][p] = c * akp - s * akq;
                a[k][q] = s * akp + c * akq;
            }
            for (int k = 0; k < 3; ++k) {   // J^T (A J)
                const double apk = a[p][k], aqk = a[q][k];
                a[p][k] = c * apk - s * aqk;
                a[q][k] = s * apk + c * aqk;
            }
            a[p][q] = a[q][p] = 0.0;
            for (int k = 0; k < 3; ++k) {   // V J
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = c * vkp - s * vkq;
                V[k][q] = s * vkp + c * vkq;
            }
        }
    }
    for (int k = 0; k < 3; ++k) w[k] = a[k][k];
}

// out[i][j] = sum_k V[i][k] d[k] V[j][k]  (= V diag(d) V^T, row-major 9 values)
__host__ __device__ __forceinline__ void sym3_compose(const double (&V)[3][3], const double (&d)[3], double* out) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) out[i * 3 + j] = V[i][0] * d[0] * V[j][0] + V[i][1] * d[1] * V[j][1] + V[i][2] * d[2] * V[j][2];
}

}  // namespace

// Finite-difference Hessians, dipole and polarizability derivatives from batched displaced-force evaluations (the scheme
// of ASE's Vibrations / Infrared, which the reference's users reach through SpkCalculator; layouts of the reference's
// atomistic.Response, nn/utils.py:21-126).
//
// The B-system batch is replicated replica-major into C = n_cols * nfree copies (copy c = d_local * nfree + s holds the
// atoms [c N, (c+1) N) and the systems [c B, (c+1) B)).  Copy (d_local, s) displaces coordinate d = chunk * n_cols +
// d_local of every system by stencil offset s; a system with d >= 3 n_m is left undisplaced in that copy (idle).  With
// n_displaced given, only the first n_displaced[m] atoms of system m are displaced (phonons.py displaces the primitive
// atoms of a supercell) and the Hessian columns run over their coordinates only.  One
// chunk is: k_vib_displace, the model on the replica batch, k_vib_assemble.  The chunk index lives in a device counter
// pair, so one captured step serves every chunk:
//   counter[0] = the chunk the next displacement reads, counter[1] = the chunk the last displacement wrote plus one;
//   k_vib_displace writes counter[1] = counter[0] + 1, k_vib_assemble reads chunk = counter[1] - 1 and writes
//   counter[0] = counter[1].  No kernel reads a word that another thread of the same kernel writes.
//
// The derivative at 0 uses the steps that were actually taken: the fp32 displaced coordinate minus the fp32 base, which
// is exact in fp64.  At |x| ~ 10 A the fp32 rounding of x +- h moves h = 0.01 A by ~1e-5 relative, as large as the force
// noise, so the nominal h is never the divisor.  Every value is written once, by one thread, in a fixed order: no atomics,
// bitwise reproducible.
#include "common.cuh"

namespace {

constexpr int VD_T = 256;   // threads per CTA of the displacement
constexpr int VA_T = 128;   // (column, atom) threads per CTA of the assembly
constexpr int VF_T = 256;   // Hessian elements per CTA of the finish
constexpr int VF_MAX_Y = 65535;

// stencil offset s in units of h: ASE's displacements -h, +h (nfree 2) and -2h, -h, +h, +2h (nfree 4)
__device__ __forceinline__ float stencil_offset(int s, int nfree, double h) {
    const int mult = nfree == 2 ? 2 * s - 1 : (s < 2 ? s - 2 : s - 1);
    return (float)((double)mult * h);
}

// atoms of system m whose coordinates are displaced: the first n_displaced[m], or all
__device__ __forceinline__ int64_t displaced_atoms(const spk_vib_t& p, int64_t m, int64_t first) {
    return p.n_displaced ? p.n_displaced[m] : p.sys_ptr[m + 1] - first;
}

__global__ void __launch_bounds__(VD_T) k_vib_displace(spk_vib_t p) {
    SPK_PDL_ENTER();
    const int64_t t = (int64_t)blockIdx.x * VD_T + threadIdx.x;
    const int64_t chunk = p.counter[0];
    if (t == 0) p.counter[1] = chunk + 1;
    const int64_t N = p.n_atoms, B = p.n_sys, C = p.n_cols * p.nfree;
    if (t < C * N) {
        const int64_t c = t / N, a = t - c * N;
        const int64_t m = p.idx_m[a];
        const int64_t first = p.sys_ptr[m], n_m = displaced_atoms(p, m, first);
        const int64_t d = chunk * p.n_cols + c / p.nfree;
        const int k = (d < 3 * n_m && a == first + d / 3) ? (int)(d % 3) : -1;     // the displaced component, if any
        const float off = stencil_offset((int)(c % p.nfree), p.nfree, p.delta);
#pragma unroll
        for (int q = 0; q < 3; ++q) {
            const float x = p.base[3 * a + q];
            p.positions[3 * t + q] = q == k ? __fadd_rn(x, off) : x;
        }
    }
    if (t < C * B) {
        const int64_t c = t / B, m = t - c * B;
        const int64_t first = p.sys_ptr[m], n_m = displaced_atoms(p, m, first);
        const int64_t d = chunk * p.n_cols + c / p.nfree;
        double step = 0.0;
        if (d < 3 * n_m) {
            const float x = p.base[3 * (first + d / 3) + d % 3];
            const float xd = __fadd_rn(x, stencil_offset((int)(c % p.nfree), p.nfree, p.delta));
            step = (double)xd - (double)x;
        }
        p.steps[t] = step;
    }
}

// derivative at 0 of the polynomial through (t_s, y_s): sum_s w_s y_s with the Lagrange weights
// w_s = [sum_{q != s} prod_{r != s, q} (-t_r)] / prod_{r != s} (t_s - t_r)
template <int NF>
__device__ __forceinline__ void lagrange_d0(const double* t, double* w) {
#pragma unroll
    for (int s = 0; s < NF; ++s) {
        double num = 0.0, den = 1.0;
#pragma unroll
        for (int q = 0; q < NF; ++q) {
            if (q == s) continue;
            den *= t[s] - t[q];
            double prod = 1.0;
#pragma unroll
            for (int r = 0; r < NF; ++r)
                if (r != s && r != q) prod *= -t[r];
            num += prod;
        }
        w[s] = num / den;
    }
}

template <int NF>
__device__ __forceinline__ void assemble_column(const spk_vib_t& p, int64_t chunk, int64_t d_local, int64_t a) {
    const int64_t N = p.n_atoms, B = p.n_sys;
    const int64_t m = p.idx_m[a];
    const int64_t first = p.sys_ptr[m], n3 = 3 * (p.sys_ptr[m + 1] - first);
    const int64_t d = chunk * p.n_cols + d_local;
    if (d >= 3 * displaced_atoms(p, m, first)) return;                     // idle copy of this system
    double t[NF], w[NF];
    int64_t c[NF];
#pragma unroll
    for (int s = 0; s < NF; ++s) {
        c[s] = d_local * NF + s;
        t[s] = p.steps[c[s] * B + m];
    }
    lagrange_d0<NF>(t, w);
    // column d of the raw Hessian, stored transposed: h_raw[m][d][r] = -dF_r/dx_d, rows r of atom a contiguous
    double* col = p.h_raw + p.hess_ptr[m] + d * n3 + 3 * (a - first);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        double g = 0.0;
#pragma unroll
        for (int s = 0; s < NF; ++s) g += w[s] * (double)p.forces[(c[s] * N + a) * 3 + k];
        col[k] = -g;
    }
    if (a != first) return;
    // per-system outputs: element [i, comp, dir] (comp: 3 or 3x3) of the reference's derivative_from_molecular layout
    const int64_t i = first + d / 3, dir = d % 3;
    if (p.dipole && p.dipole_deriv) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            double g = 0.0;
#pragma unroll
            for (int s = 0; s < NF; ++s) g += w[s] * (double)p.dipole[(c[s] * B + m) * 3 + k];
            p.dipole_deriv[(i * 3 + k) * 3 + dir] = g;
        }
    }
    if (p.polar && p.polar_deriv) {
#pragma unroll
        for (int k = 0; k < 9; ++k) {
            double g = 0.0;
#pragma unroll
            for (int s = 0; s < NF; ++s) g += w[s] * (double)p.polar[(c[s] * B + m) * 9 + k];
            p.polar_deriv[(i * 9 + k) * 3 + dir] = g;
        }
    }
}

__global__ void __launch_bounds__(VA_T) k_vib_assemble(spk_vib_t p) {
    SPK_PDL_ENTER();
    const int64_t t = (int64_t)blockIdx.x * VA_T + threadIdx.x;
    const int64_t chunk = p.counter[1] - 1;
    if (t == 0) p.counter[0] = chunk + 1;
    if (t >= p.n_cols * p.n_atoms) return;
    const int64_t d_local = t / p.n_atoms, a = t - d_local * p.n_atoms;
    if (p.nfree == 2)
        assemble_column<2>(p, chunk, d_local, a);
    else
        assemble_column<4>(p, chunk, d_local, a);
}

// H = (H_raw + H_raw^T) / 2 per system, written in the Response layout [n^2, 3, 3] (row i n + j, block [a, b] =
// d2E / dR_ia dR_jb) and mass-weighted [3n, 3n] times mw_scale / sqrt(m_i m_j)
__global__ void __launch_bounds__(VF_T) k_vib_finish(spk_vib_t p) {
    SPK_PDL_ENTER();
    const int64_t e = (int64_t)blockIdx.x * VF_T + threadIdx.x;
    for (int64_t m = blockIdx.y; m < p.n_sys; m += gridDim.y) {
        const int64_t first = p.sys_ptr[m], n = p.sys_ptr[m + 1] - first, n3 = 3 * n;
        if (e >= n3 * n3) continue;
        const int64_t b = e % 3, a = (e / 3) % 3, ij = e / 9, i = ij / n, j = ij - i * n;
        const int64_t r = 3 * i + a, c = 3 * j + b;
        const double* raw = p.h_raw + p.hess_ptr[m];
        const double h = 0.5 * (raw[c * n3 + r] + raw[r * n3 + c]);
        p.hessian[p.hess_ptr[m] + e] = h;
        p.hessian_mw[p.hess_ptr[m] + r * n3 + c] =
            h * p.mw_scale / sqrt(p.masses[first + i] * p.masses[first + j]);
    }
}

int check_params(const spk_vib_t* p) {
    if (!p || p->n_atoms < 0 || p->n_sys < 1 || p->n_cols < 1 || (p->nfree != 2 && p->nfree != 4)) return SPK_ERR_ARG;
    if (!(p->delta > 0.0) || !p->sys_ptr || !p->hess_ptr || !p->counter) return SPK_ERR_ARG;
    return SPK_OK;
}

}  // namespace

extern "C" int spk_vib_displace(const spk_vib_t* p, spk_stream_t stream) {
    if (check_params(p) != SPK_OK || !p->base || !p->positions || !p->steps || (p->n_atoms > 0 && !p->idx_m))
        return SPK_ERR_ARG;
    const int64_t C = p->n_cols * p->nfree;
    const int64_t n = C * (p->n_atoms > p->n_sys ? p->n_atoms : p->n_sys);
    spk_launch(k_vib_displace, (unsigned)spk_cdiv(n, VD_T), VD_T, 0, spk_st(stream), *p);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_vib_assemble(const spk_vib_t* p, spk_stream_t stream) {
    if (check_params(p) != SPK_OK || !p->steps || !p->h_raw || (p->n_atoms > 0 && (!p->idx_m || !p->forces)))
        return SPK_ERR_ARG;
    if ((p->dipole_deriv && !p->dipole) || (p->polar_deriv && !p->polar)) return SPK_ERR_ARG;
    const int64_t n = p->n_cols * p->n_atoms;
    spk_launch(k_vib_assemble, (unsigned)(n > 0 ? spk_cdiv(n, VA_T) : 1), VA_T, 0, spk_st(stream), *p);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_vib_finish(const spk_vib_t* p, spk_stream_t stream) {
    if (check_params(p) != SPK_OK || !p->h_raw || !p->hessian || !p->hessian_mw || (p->n_atoms > 0 && !p->masses) ||
        p->max_atoms < 0 || p->n_displaced)         // the finish symmetrises square blocks: every atom displaced
        return SPK_ERR_ARG;
    const int64_t n3 = 3 * p->max_atoms;
    if (n3 == 0) return SPK_OK;
    const dim3 grid((unsigned)spk_cdiv(n3 * n3, VF_T), (unsigned)(p->n_sys < VF_MAX_Y ? p->n_sys : VF_MAX_Y));
    spk_launch(k_vib_finish, grid, VF_T, 0, spk_st(stream), *p);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

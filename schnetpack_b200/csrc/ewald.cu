// Reciprocal-space and self terms of the Ewald sum (atomistic/electrostatic.py:310-375); the real-space term is a kind of
// pair_energy.cu.  Per system m with cell h, H = h^-1, V = |det h| and k = 2 pi n H^T for the integer triples n:
//   E_rec = ke (2 pi / V) sum_k f_k |S_k|^2,  f_k = exp(-k^2 / (4 alpha)) / k^2,  S_k = sum_i q_i e^{i k.r_i}
//   E_self = ke sqrt(alpha / pi) sum_i q_i^2
// Phases: k.r_i = 2 pi n.s_i with the fractional coordinates s_i = r_i H, reduced mod 1 in fp64 (exact for integer n), so
// sincospi sees arguments of a few times k_max whatever the unwrapped positions are.
//
// Layout.  Forward: one thread per (system, k-vector) sums over the system's atoms, staged EW_T at a time in shared
// memory, and keeps a record (k, f_k, S_k) per (system, k) in the workspace; one CTA per system then sums f_k |S_k|^2 and
// q_i^2 in a fixed strided order and a fixed tree.  Reverse: one CTA per (system, tile of up to EW_T atoms) runs over the
// k-vectors of that system, staged EW_T at a time, with the lanes of a small tile sharing each atom's k-vectors; the k
// range is split over grid.y so that a box of a few thousand atoms still fills the GPU, and a second pass adds the splits
// in order.  That pass also forms r_i (x) g_R_i and hands it to the segmented-partial pass
// of segscan.cuh; one CTA per system finishes it and the k-sums of the cell gradient and the virial.  No atomics anywhere:
// every result is bitwise the same on every call.  Cost: N K complex terms per direction, each one fp64 sincospi and a
// handful of fp64 FMAs, so the kernels are bound by the fp64 pipe.
#include <math.h>

#include "common.cuh"
#include "segscan.cuh"
#include "ewald_common.cuh"

namespace {

constexpr int EW_T = 128;            // k-vectors per CTA (forward), atoms per CTA (reverse), staging tile of both
constexpr int EW_KREC = 6;           // doubles per (system, k) record: k [3], f_k, Re S_k, Im S_k
constexpr int EW_SPLIT_K = 1024;     // k-vectors per split of the reverse (at least)
constexpr int EW_MAX_SPLIT = 64;

static_assert(EW_T == SEG_FIN_T, "the per-system passes reuse the partial layout of EW_T-item CTAs");

inline int64_t ew_splits(int64_t n_k) {
    const int64_t s = n_k / EW_SPLIT_K;
    return s < 1 ? 1 : (s > EW_MAX_SPLIT ? EW_MAX_SPLIT : s);
}

inline int64_t ew_split_len(int64_t n_k) { return spk_cdiv(spk_cdiv(n_k, ew_splits(n_k)), EW_T) * EW_T; }

struct EwLayout {
    double *sys, *frac, *krec, *apart, *part;
    int64_t n_split;
};

inline size_t ew_doubles(int64_t N, int64_t B, int64_t K, EwLayout* L, double* base) {
    const int64_t ns = ew_splits(K);
    const int64_t nb = spk_cdiv(N, EW_T);
    const int64_t n_sys_rec = EW_SYS * B, n_frac = 3 * N, n_krec = EW_KREC * B * K, n_apart = 4 * ns * N;
    const int64_t n_part = 9 * (B + nb + 1);
    if (L) {
        L->sys = base;
        L->frac = L->sys + n_sys_rec;
        L->krec = L->frac + n_frac;
        L->apart = L->krec + n_krec;
        L->part = L->apart + n_apart;
        L->n_split = ns;
    }
    return (size_t)(n_sys_rec + n_frac + n_krec + n_apart + n_part);
}

__device__ __forceinline__ void k_of(const double* __restrict__ H, double n0, double n1, double n2, double& kx,
                                     double& ky, double& kz) {
    kx = 2.0 * EW_PI * (n0 * H[0] + n1 * H[1] + n2 * H[2]);
    ky = 2.0 * EW_PI * (n0 * H[3] + n1 * H[4] + n2 * H[5]);
    kz = 2.0 * EW_PI * (n0 * H[6] + n1 * H[7] + n2 * H[8]);
}

// S_k of system blockIdx.y for the k-vectors of CTA blockIdx.x, and the record (k, f_k, S_k)
__global__ void __launch_bounds__(EW_T) k_ewald_sk(const float* __restrict__ q, const double* __restrict__ frac,
                                                   const float* __restrict__ kvecs, const int32_t* __restrict__ sys_ptr,
                                                   const double* __restrict__ sys, int64_t n_k, double alpha,
                                                   double* __restrict__ krec) {
    __shared__ double st[EW_T][4];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t m = blockIdx.y;
    const int64_t k = (int64_t)blockIdx.x * EW_T + t;
    const bool valid = k < n_k;
    const double n0 = valid ? kvecs[3 * k] : 0.0, n1 = valid ? kvecs[3 * k + 1] : 0.0, n2 = valid ? kvecs[3 * k + 2] : 0.0;
    const int64_t a0 = sys_ptr[m], a1 = sys_ptr[m + 1];
    double re = 0.0, im = 0.0;
    for (int64_t base = a0; base < a1; base += EW_T) {
        const int cnt = (int)min((int64_t)EW_T, a1 - base);
        __syncthreads();
        if (t < cnt) {
            const int64_t a = base + t;
            st[t][0] = frac[3 * a], st[t][1] = frac[3 * a + 1], st[t][2] = frac[3 * a + 2], st[t][3] = q[a];
        }
        __syncthreads();
        for (int j = 0; j < cnt; ++j) {
            double sn, cs;
            sincospi(2.0 * (n0 * st[j][0] + n1 * st[j][1] + n2 * st[j][2]), &sn, &cs);
            re = fma(st[j][3], cs, re);
            im = fma(st[j][3], sn, im);
        }
    }
    if (!valid) return;
    double kx, ky, kz;
    k_of(sys + EW_SYS * m, n0, n1, n2, kx, ky, kz);
    const double k2 = kx * kx + ky * ky + kz * kz;
    double* r = krec + EW_KREC * (m * n_k + k);
    r[0] = kx, r[1] = ky, r[2] = kz, r[3] = exp(-0.25 * k2 / alpha) / k2, r[4] = re, r[5] = im;
}

// energy[m] = addend[m] + ke ((2 pi / V) sum_k f_k |S_k|^2 - sqrt(alpha / pi) sum_i q_i^2)
__global__ void __launch_bounds__(SEG_FIN_T) k_ewald_energy(const float* __restrict__ q,
                                                            const int32_t* __restrict__ sys_ptr,
                                                            const double* __restrict__ sys,
                                                            const double* __restrict__ krec, int64_t n_k, double ke,
                                                            double alpha, const float* __restrict__ addend,
                                                            float* __restrict__ energy) {
    __shared__ double red[2][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t m = blockIdx.x;
    double acc[2] = {0.0, 0.0};
    for (int64_t k = t; k < n_k; k += SEG_FIN_T) {
        const double* r = krec + EW_KREC * (m * n_k + k);
        acc[0] += r[3] * (r[4] * r[4] + r[5] * r[5]);
    }
    for (int64_t a = sys_ptr[m] + t; a < sys_ptr[m + 1]; a += SEG_FIN_T) acc[1] += (double)q[a] * (double)q[a];
    ew_tree<2>(acc, red);
    if (t != 0) return;
    const double V = sys[EW_SYS * m + 9];
    double e = ke * (2.0 * EW_PI / V * red[0][0] - sqrt(alpha / EW_PI) * red[1][0]);
    if (!(V > 0.0)) e = __longlong_as_double(0x7ff8000000000000ll);     // zero volume: the reference raises
    energy[m] = (float)((addend ? (double)addend[m] : 0.0) + e);
}

// First CTA of system m in the (system, atom-tile) grid of the reverse: sys_ptr[m] / EW_T + m.  Consecutive starts differ
// by at least max(1, cdiv(n_m, EW_T)) CTAs, so every system gets its tiles of EW_T atoms, no CTA holds two systems, and
// the grid has N / EW_T + n_sys CTAs (a shape that depends on N and n_sys only).
__device__ __forceinline__ int64_t ew_tile0(const int32_t* __restrict__ sys_ptr, int64_t m) {
    return sys_ptr[m] / EW_T + m;
}

// Per (atom, k-split): sum over the split's k-vectors of the atom's system of 2 f_k k (Im S cos - Re S sin) [3] and
// 2 f_k (Re S cos + Im S sin).  A CTA holds one tile of up to EW_T atoms of one system; G = EW_T / pow2ceil(n_tile)
// consecutive lanes share an atom and take every G-th staged k-vector, so a tile of a small system still keeps every lane
// busy.  The G lane sums of an atom are added in lane order.
__global__ void __launch_bounds__(EW_T) k_ewald_atom_k(const double* __restrict__ frac, const float* __restrict__ kvecs,
                                                       const int32_t* __restrict__ sys_ptr, const double* __restrict__ krec,
                                                       int64_t n_sys, int64_t n_atoms, int64_t n_k, int64_t split_len,
                                                       double* __restrict__ apart) {
    __shared__ double st[EW_T][8];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t b = blockIdx.x;
    int64_t lo = 0, hi = n_sys - 1;                  // the system whose tiles hold CTA b
    while (lo < hi) {
        const int64_t mid = (lo + hi + 1) >> 1;
        if (ew_tile0(sys_ptr, mid) <= b) lo = mid;
        else hi = mid - 1;
    }
    const int64_t m = lo;
    const int64_t a0 = sys_ptr[m] + (b - ew_tile0(sys_ptr, m)) * EW_T, a1 = sys_ptr[m + 1];
    if (a0 >= a1) return;                            // a spare tile: the whole CTA leaves
    const int na = (int)min((int64_t)EW_T, a1 - a0);
    int p2 = 1;
    while (p2 < na) p2 <<= 1;
    const int G = EW_T / p2;
    const int ai = t / G, lane = t - ai * G;
    const bool active = ai < na;
    const int64_t a = a0 + ai;
    const int64_t k0 = (int64_t)blockIdx.y * split_len, k1 = min(k0 + split_len, n_k);
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    if (active) s0 = frac[3 * a], s1 = frac[3 * a + 1], s2 = frac[3 * a + 2];
    double gx = 0.0, gy = 0.0, gz = 0.0, gq = 0.0;
    for (int64_t kb = k0; kb < k1; kb += EW_T) {
        const int cnt = (int)min((int64_t)EW_T, k1 - kb);
        __syncthreads();
        if (t < cnt) {
            const int64_t k = kb + t;
            const double* r = krec + EW_KREC * (m * n_k + k);
            const double f2 = 2.0 * r[3];
            st[t][0] = kvecs[3 * k], st[t][1] = kvecs[3 * k + 1], st[t][2] = kvecs[3 * k + 2];
            st[t][3] = r[0], st[t][4] = r[1], st[t][5] = r[2], st[t][6] = f2 * r[4], st[t][7] = f2 * r[5];
        }
        __syncthreads();
        if (!active) continue;
#pragma unroll 4
        for (int j = lane; j < cnt; j += G) {
            double sn, cs;
            sincospi(2.0 * (st[j][0] * s0 + st[j][1] * s1 + st[j][2] * s2), &sn, &cs);
            const double u = st[j][7] * cs - st[j][6] * sn;
            gx = fma(u, st[j][3], gx);
            gy = fma(u, st[j][4], gy);
            gz = fma(u, st[j][5], gz);
            gq = fma(st[j][6], cs, fma(st[j][7], sn, gq));
        }
    }
    __syncthreads();
    st[t][0] = gx, st[t][1] = gy, st[t][2] = gz, st[t][3] = gq;
    __syncthreads();
    if (!active || lane != 0) return;
    double g[4] = {0.0, 0.0, 0.0, 0.0};
    for (int u = 0; u < G; ++u) {
#pragma unroll
        for (int c = 0; c < 4; ++c) g[c] += st[t + u][c];
    }
    double* o = apart + 4 * ((int64_t)blockIdx.y * n_atoms + a);
    o[0] = g[0], o[1] = g[1], o[2] = g[2], o[3] = g[3];
}

// g_R, g_q of each atom from the splits (added in split order), and the partials of sum_i r_i (x) g_R_i per system
__global__ void __launch_bounds__(EW_T) k_ewald_atom_fin(const float* __restrict__ R, const float* __restrict__ q,
                                                         const int64_t* __restrict__ idx_m,
                                                         const int32_t* __restrict__ sys_ptr,
                                                         const double* __restrict__ sys, const double* __restrict__ apart,
                                                         int64_t n_atoms, int64_t n_split, double ke, double alpha,
                                                         const float* __restrict__ g_E, float* __restrict__ g_R,
                                                         float* __restrict__ g_q, int accumulate_q,
                                                         double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * EW_T + threadIdx.x;
    double v[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) v[c] = 0.0;
    int64_t m = 0, first = 0, end = 0;
    if (a < n_atoms) {
        m = idx_m[a];
        first = sys_ptr[m];
        end = sys_ptr[m + 1];
        double g[4] = {0.0, 0.0, 0.0, 0.0};
        for (int64_t s = 0; s < n_split; ++s) {
            const double* o = apart + 4 * (s * n_atoms + a);
#pragma unroll
            for (int c = 0; c < 4; ++c) g[c] += o[c];
        }
        const double gE = g_E[m], qa = q[a];
        const double pre = ke * 2.0 * EW_PI / sys[EW_SYS * m + 9];
        const double gR[3] = {pre * gE * qa * g[0], pre * gE * qa * g[1], pre * gE * qa * g[2]};
        if (g_R) {
#pragma unroll
            for (int c = 0; c < 3; ++c) g_R[3 * a + c] = (float)gR[c];
        }
        if (g_q) {
            const double gq = gE * (pre * g[3] - 2.0 * ke * sqrt(alpha / EW_PI) * qa);
            g_q[a] = (float)((accumulate_q ? (double)g_q[a] : 0.0) + gq);
        }
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            const double r = R[3 * a + b];
#pragma unroll
            for (int c = 0; c < 3; ++c) v[3 * b + c] = r * gR[c];
        }
    }
    seg_partials<EW_T, 9>(v, n_atoms, m, first, end, sys_part, head);
}

// Per system: T = sum_k E_k (1/k^2 + 1/(4 alpha)) k (x) k and E_rec, then g_cell = -H^T [sum_i r_i (x) g_R_i - 2 g_E T +
// g_E E_rec I] and the virial -g_E (E_rec I - 2 T)
__global__ void __launch_bounds__(SEG_FIN_T) k_ewald_sys_bwd(const int32_t* __restrict__ sys_ptr,
                                                             const double* __restrict__ sys,
                                                             const double* __restrict__ krec, int64_t n_k, double ke,
                                                             double alpha, const float* __restrict__ g_E,
                                                             const double* __restrict__ sys_part,
                                                             const double* __restrict__ head, float* __restrict__ g_cell,
                                                             double* __restrict__ virial, int accumulate_virial) {
    __shared__ double red[9][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t m = blockIdx.x;
    double acc[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int64_t k = t; k < n_k; k += SEG_FIN_T) {
        const double* r = krec + EW_KREC * (m * n_k + k);
        const double kx = r[0], ky = r[1], kz = r[2];
        const double e = r[3] * (r[4] * r[4] + r[5] * r[5]);
        const double w = e * (1.0 / (kx * kx + ky * ky + kz * kz) + 0.25 / alpha);
        acc[0] += e;
        acc[1] += w * kx * kx, acc[2] += w * ky * ky, acc[3] += w * kz * kz;
        acc[4] += w * kx * ky, acc[5] += w * kx * kz, acc[6] += w * ky * kz;
    }
    ew_tree<7>(acc, red);
    double tot[7];
#pragma unroll
    for (int c = 0; c < 7; ++c) tot[c] = red[c][0];
    __syncthreads();
    seg_finish_block<EW_T, 9>(sys_ptr, nullptr, sys_part, head, m, red);
    if (t != 0) return;
    const double* H = sys + EW_SYS * m;
    const double c = ke * 2.0 * EW_PI / H[9];
    const double gE = g_E[m];
    const double E = c * tot[0];
    const double T[9] = {c * tot[1], c * tot[4], c * tot[5], c * tot[4], c * tot[2], c * tot[6],
                         c * tot[5], c * tot[6], c * tot[3]};
    if (g_cell) {
        double M[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) M[i] = red[i][0] - 2.0 * gE * T[i] + (i % 4 == 0 ? gE * E : 0.0);
#pragma unroll
        for (int b = 0; b < 3; ++b) {
#pragma unroll
            for (int d = 0; d < 3; ++d)
                g_cell[9 * m + 3 * b + d] = (float)-(H[b] * M[d] + H[3 + b] * M[3 + d] + H[6 + b] * M[6 + d]);
        }
    }
    if (virial) {
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            const double w = -gE * ((i % 4 == 0 ? E : 0.0) - 2.0 * T[i]);
            virial[9 * m + i] = accumulate_virial ? virial[9 * m + i] + w : w;
        }
    }
}

}  // namespace

extern "C" size_t spk_ewald_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n_k) {
    if (n_atoms < 0 || n_sys < 0 || n_k < 0) return 0;
    return sizeof(double) * ew_doubles(n_atoms, n_sys, n_k, nullptr, nullptr);
}

static int ew_check(const float* R, const float* q, const float* cell, const float* kvecs, const int64_t* idx_m,
                    const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int64_t n_k, double alpha, void* workspace,
                    size_t workspace_bytes) {
    if (n_atoms < 0 || n_sys < 0 || n_k < 0 || n_atoms >= (1ll << 31) - 1 || n_sys > 65535) return SPK_ERR_ARG;
    if (!(alpha > 0.0)) return SPK_ERR_ARG;
    if (n_sys == 0) return SPK_OK;
    if (!cell || !sys_ptr || !workspace || (n_k > 0 && !kvecs)) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!R || !q || !idx_m)) return SPK_ERR_ARG;
    if (workspace_bytes < spk_ewald_workspace_bytes(n_atoms, n_sys, n_k)) return SPK_ERR_ARG;
    return SPK_OK;
}

extern "C" int spk_ewald_fwd(const float* R, const float* q, const float* cell, const float* kvecs,
                             const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int64_t n_k,
                             double ke, double alpha, const float* addend, float* energy, void* workspace,
                             size_t workspace_bytes, spk_stream_t stream) {
    const int rc = ew_check(R, q, cell, kvecs, idx_m, sys_ptr, n_atoms, n_sys, n_k, alpha, workspace, workspace_bytes);
    if (rc != SPK_OK || n_sys == 0) return rc;
    if (!energy) return SPK_ERR_ARG;
    EwLayout L;
    ew_doubles(n_atoms, n_sys, n_k, &L, reinterpret_cast<double*>(workspace));
    const cudaStream_t st = spk_st(stream);
    spk_launch(k_ewald_cell, (unsigned)spk_cdiv(n_sys, 128), 128, 0, st, cell, n_sys, L.sys);
    if (n_atoms > 0)
        spk_launch(k_ewald_frac, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, R, idx_m, L.sys, n_atoms, L.frac);
    if (n_k > 0)
        spk_launch(k_ewald_sk, dim3((unsigned)spk_cdiv(n_k, EW_T), (unsigned)n_sys), EW_T, 0, st, q, L.frac, kvecs,
                   sys_ptr, L.sys, n_k, alpha, L.krec);
    spk_launch(k_ewald_energy, (unsigned)n_sys, SEG_FIN_T, 0, st, q, sys_ptr, L.sys, L.krec, n_k, ke, alpha, addend,
               energy);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_ewald_bwd(const float* R, const float* q, const float* cell, const float* kvecs,
                             const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int64_t n_k,
                             double ke, double alpha, const float* g_E, float* g_R, float* g_q, int accumulate_q,
                             float* g_cell, double* virial, int accumulate_virial, void* workspace,
                             size_t workspace_bytes, spk_stream_t stream) {
    const int rc = ew_check(R, q, cell, kvecs, idx_m, sys_ptr, n_atoms, n_sys, n_k, alpha, workspace, workspace_bytes);
    if (rc != SPK_OK || n_sys == 0) return rc;
    if (!g_E) return SPK_ERR_ARG;
    EwLayout L;
    ew_doubles(n_atoms, n_sys, n_k, &L, reinterpret_cast<double*>(workspace));
    const cudaStream_t st = spk_st(stream);
    const int64_t nb = spk_cdiv(n_atoms, EW_T);
    double* sys_part = L.part;
    double* head = sys_part + 9 * n_sys;
    if (n_atoms > 0) {
        if (n_k > 0)
            spk_launch(k_ewald_atom_k, dim3((unsigned)(n_atoms / EW_T + n_sys), (unsigned)L.n_split), EW_T, 0, st, L.frac,
                       kvecs, sys_ptr, L.krec, n_sys, n_atoms, n_k, ew_split_len(n_k), L.apart);
        spk_launch(k_ewald_atom_fin, (unsigned)nb, EW_T, 0, st, R, q, idx_m, sys_ptr, L.sys, L.apart, n_atoms,
                   n_k > 0 ? L.n_split : (int64_t)0, ke, alpha, g_E, g_R, g_q, accumulate_q, sys_part, head);
    }
    if (g_cell || virial)
        spk_launch(k_ewald_sys_bwd, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, L.sys, L.krec, n_k, ke, alpha, g_E,
                   sys_part, head, g_cell, virial, accumulate_virial);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

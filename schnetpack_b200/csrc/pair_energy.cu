// Pair energies of the physics add-ons: ZBL nuclear repulsion (atomistic/nuclear_repulsion.py:81-104), the Coulomb
// energy of point charges, plain or damped and optionally shifted to zero at a cutoff (atomistic/electrostatic.py:14-152),
// and the real-space term of the Ewald sum (atomistic/electrostatic.py:266-308; the reciprocal and self terms are in
// ewald.cu).
//
// Per edge e = (i, j) with d = |r_ij| the term e_ij is evaluated in fp64 from the fp32 inputs; per system the energy is
// 0.5 ke sum_{e in m} e_ij.  The edges of system m are the receiver slots [rowptr[sys_ptr[m]], rowptr[sys_ptr[m+1]]), the
// mapping of spk_pairwise_virial, and the two passes of segscan.cuh sum them (seg_partials over PE_T consecutive slots,
// then a per-system finish), so the energies are bitwise the same on every call, without atomics, for any mix of system
// sizes.  The reverse recomputes the terms instead of keeping a tape: g_rij is elementwise in edge order, and the charge
// gradient of the Coulomb term is a per-atom sum over the atom's receiver slots, then its sender slots, in the fixed CSR
// order of the two graph views.
#include <math.h>

#include "common.cuh"
#include "segscan.cuh"

namespace {

constexpr int PE_T = 256;

__device__ __forceinline__ double softplus_d(double x) { return x > 20.0 ? x : log1p(exp(x)); }   // F.softplus

// ZBL screened repulsion (nuclear_repulsion.py:81-99) times the optional cosine cutoff (nn/cutoff.py:14-33): e and de/dd.
// The parameters are read raw from device memory and softplus / L1 normalisation are applied here, so that a captured
// graph sees updated parameter values.
__device__ __forceinline__ void zbl_term(const spk_pair_t& p, double d, double zi, double zj, double& e, double& de) {
    const int K = p.n_terms;
    const double pw = softplus_d((double)p.a_pow[0]);
    const double adiv = softplus_d((double)p.a_div[0]);
    double csum = 0.0;
    for (int k = 0; k < K; ++k) csum += fabs(softplus_d((double)p.coefficients[k]));
    csum = fmax(csum, 1e-12);                                                    // F.normalize(p=1, eps=1e-12)
    const double aij = (pow(zi, pw) + pow(zj, pw)) * adiv;
    double scr = 0.0, dscr = 0.0;
    for (int k = 0; k < K; ++k) {
        const double c = softplus_d((double)p.coefficients[k]) / csum;
        const double a = aij * softplus_d((double)p.exponents[k]);
        const double x = c * exp(-a * d);
        scr += x;
        dscr -= a * x;
    }
    const double rep = zi * zj / d, drep = -rep / d;
    double fc = 1.0, dfc = 0.0;
    if (p.cutoff > 0.0) {
        const double w = M_PI / p.cutoff;
        fc = d < p.cutoff ? 0.5 * (cos(w * d) + 1.0) : 0.0;
        dfc = d < p.cutoff ? -0.5 * w * sin(w * d) : 0.0;
    }
    e = rep * fc * scr;
    de = drep * fc * scr + rep * dfc * scr + rep * fc * dscr;
}

// exp(-1/y) for y > 0, else 0 (nn/cutoff.py:107-122), and its derivative
__device__ __forceinline__ void switch_component(double y, double& f, double& df) {
    if (y <= 0.0) {
        f = 0.0, df = 0.0;
    } else {
        f = exp(-1.0 / y);
        df = f / (y * y);
    }
}

// SwitchFunction of (switch_on, switch_off) (nn/cutoff.py:125-158): 1 below switch_on, 0 above switch_off, and its
// derivative
__device__ __forceinline__ void switch_function(const spk_pair_t& p, double d, double& sw, double& dsw) {
    const double w = p.switch_off - p.switch_on;
    const double x = (d - p.switch_on) / w;
    sw = 1.0, dsw = 0.0;
    if (x >= 1.0) {
        sw = 0.0;
    } else if (x > 0.0) {
        double fp, dfp, fm, dfm;
        switch_component(x, fp, dfp);
        switch_component(1.0 - x, fm, dfm);
        dfm = -dfm;
        const double den = fp + fm;
        sw = fm / den;
        dsw = (dfm * fp - fm * dfp) / (den * den) / w;
    }
}

// Ewald real-space potential (electrostatic.py:292-300) V = erfc(sqrt(alpha) d) / d, times 1 - screen(d) when a
// SwitchFunction screen is given (switch_off != switch_on), and dV/dd.  No cutoff: every pair of the list counts.
__device__ __forceinline__ void ewald_real_potential(const spk_pair_t& p, double d, double& V, double& dV) {
    const double a = sqrt(p.alpha);
    const double inv = 1.0 / d;
    const double ec = erfc(a * d);
    V = ec * inv;
    dV = -(1.1283791670955126 * a * exp(-a * a * d * d) + V) * inv;    // 2 / sqrt(pi)
    if (p.switch_off != p.switch_on) {
        double sw, dsw;
        switch_function(p, d, sw, dsw);
        dV = dV * (1.0 - sw) - V * dsw;
        V = V * (1.0 - sw);
    }
}

// Coulomb potential V(d) and dV/dd: 1/d or the damped form of electrostatic.py:43-57 with SwitchFunction
// (nn/cutoff.py:125-158), shifted to zero at the cutoff (electrostatic.py:141-145).
__device__ __forceinline__ void coulomb_potential(const spk_pair_t& p, double d, double& V, double& dV) {
    const double inv = 1.0 / d;
    V = inv;
    dV = -inv * inv;
    if (p.kind == SPK_PAIR_DAMPED_COULOMB) {
        double sw, dsw;
        switch_function(p, d, sw, dsw);
        const double r2 = d * d + 1.0;
        const double damped = 1.0 / sqrt(r2);
        V = sw * damped + (1.0 - sw) * inv;
        dV = dsw * (damped - inv) - sw * d * damped / r2 - (1.0 - sw) * inv * inv;
    }
    if (p.cutoff > 0.0) {
        if (d <= p.cutoff) {
            const double s2 = p.shift * p.shift;
            dV = dV * (1.0 - s2 / (V * V));
            V = V + s2 / V - 2.0 * p.shift;
        } else {
            V = 0.0, dV = 0.0;
        }
    }
}

// the potential of a charge-pair kind: Coulomb, damped Coulomb or the Ewald real-space term
__device__ __forceinline__ void charge_potential(const spk_pair_t& p, double d, double& V, double& dV) {
    if (p.kind == SPK_PAIR_EWALD_REAL) ewald_real_potential(p, d, V, dV);
    else coulomb_potential(p, d, V, dV);
}

__device__ __forceinline__ bool masked(const spk_pair_t& p, double d) { return p.d_max > 0.0 && !(d <= p.d_max); }

__device__ __forceinline__ double edge_distance(const float* __restrict__ r) {
    const double x = r[0], y = r[1], z = r[2];
    return sqrt(x * x + y * y + z * z);
}

// e_ij, de/dd and (Coulomb) the potential V of edge e between atoms i and j
__device__ __forceinline__ void pair_term(const spk_pair_t& p, double d, const int64_t* __restrict__ Z,
                                          const float* __restrict__ q, int64_t i, int64_t j, double& e, double& de,
                                          double& V) {
    e = 0.0, de = 0.0, V = 0.0;
    if (masked(p, d) || !(d > 0.0)) return;
    if (p.kind == SPK_PAIR_ZBL) {
        zbl_term(p, d, (double)Z[i], (double)Z[j], e, de);
    } else {
        double dV;
        charge_potential(p, d, V, dV);
        const double qq = (double)q[i] * (double)q[j];
        e = qq * V;
        de = qq * dV;
    }
}

__global__ void __launch_bounds__(PE_T) k_pair_partials(spk_pair_t p, const float* __restrict__ r_ij,
                                                        const int64_t* __restrict__ idx_i, const int64_t* __restrict__ idx_j,
                                                        const int64_t* __restrict__ Z, const float* __restrict__ q,
                                                        const int64_t* __restrict__ idx_m, const int32_t* __restrict__ rowptr,
                                                        const int32_t* __restrict__ slot_eid,
                                                        const int32_t* __restrict__ sys_ptr, int64_t n_sys,
                                                        double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t s = (int64_t)blockIdx.x * PE_T + threadIdx.x;
    const int64_t n_slots = rowptr[sys_ptr[n_sys]];
    double v[1] = {0.0};
    int64_t m = 0, first = 0, end = 0;
    if (s < n_slots) {
        const int64_t e = slot_eid[s];
        const int64_t i = idx_i[e];
        double de, V;
        pair_term(p, edge_distance(r_ij + 3 * e), Z, q, i, idx_j[e], v[0], de, V);
        m = idx_m[i];
        first = rowptr[sys_ptr[m]];
        end = rowptr[sys_ptr[m + 1]];
    }
    seg_partials<PE_T, 1>(v, n_slots, m, first, end, sys_part, head);
}

__global__ void __launch_bounds__(SEG_FIN_T) k_pair_finish(const int32_t* __restrict__ rowptr,
                                                           const int32_t* __restrict__ sys_ptr,
                                                           const double* __restrict__ sys_part,
                                                           const double* __restrict__ head, double scale,
                                                           float* __restrict__ energy) {
    __shared__ double red[1][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t m = blockIdx.x;
    seg_finish_block<PE_T, 1>(rowptr, sys_ptr, sys_part, head, m, red);
    if (threadIdx.x == 0) energy[m] = (float)(scale * red[0][0]);
}

// g_rij[e] = 0.5 ke g_E[m(e)] de/dd r_ij / d, in edge order
__global__ void k_pair_grad_rij(spk_pair_t p, const float* __restrict__ r_ij, const int64_t* __restrict__ idx_i,
                                const int64_t* __restrict__ idx_j, const int64_t* __restrict__ Z, const float* __restrict__ q,
                                const int64_t* __restrict__ idx_m, const float* __restrict__ g_E, int64_t n_edges,
                                double scale, float* __restrict__ g_rij) {
    SPK_PDL_ENTER();
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= n_edges) return;
    const float* r = r_ij + 3 * e;
    const double d = edge_distance(r);
    const int64_t i = idx_i[e];
    double en, de, V;
    pair_term(p, d, Z, q, i, idx_j[e], en, de, V);
    const double f = de != 0.0 ? scale * (double)g_E[idx_m[i]] * de / d : 0.0;
    g_rij[3 * e] = (float)(f * r[0]);
    g_rij[3 * e + 1] = (float)(f * r[1]);
    g_rij[3 * e + 2] = (float)(f * r[2]);
}

// g_q[a] = 0.5 ke g_E[m(a)] (sum_{receiver slots of a} q_j V + sum_{sender slots of a} q_i V), fp64 in CSR order
__global__ void k_pair_grad_q(spk_pair_t p, const float* __restrict__ r_ij, const float* __restrict__ q,
                              const int64_t* __restrict__ idx_m, const float* __restrict__ g_E,
                              const int32_t* __restrict__ rowptr, const int32_t* __restrict__ slot_j,
                              const int32_t* __restrict__ slot_eid, const int32_t* __restrict__ sptr,
                              const int32_t* __restrict__ pos_slot, const int32_t* __restrict__ pos_i, int64_t n_atoms,
                              double scale, float* __restrict__ g_q) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    double acc = 0.0, de, V;
    for (int64_t s = rowptr[a]; s < rowptr[a + 1]; ++s) {
        const int64_t e = slot_eid[s];
        const double d = edge_distance(r_ij + 3 * e);
        if (masked(p, d) || !(d > 0.0)) continue;
        charge_potential(p, d, V, de);
        acc += (double)q[slot_j[s]] * V;
    }
    for (int64_t k = sptr[a]; k < sptr[a + 1]; ++k) {
        const int64_t e = slot_eid[pos_slot[k]];
        const double d = edge_distance(r_ij + 3 * e);
        if (masked(p, d) || !(d > 0.0)) continue;
        charge_potential(p, d, V, de);
        acc += (double)q[pos_i[k]] * V;
    }
    g_q[a] = (float)(scale * (double)g_E[idx_m[a]] * acc);
}

int check_pair(const spk_pair_t* p) {
    if (!p) return SPK_ERR_ARG;
    if (p->kind != SPK_PAIR_ZBL && p->kind != SPK_PAIR_COULOMB && p->kind != SPK_PAIR_DAMPED_COULOMB &&
        p->kind != SPK_PAIR_EWALD_REAL)
        return SPK_ERR_ARG;
    if (p->kind == SPK_PAIR_ZBL) {
        if (p->n_terms <= 0 || p->n_terms > SPK_PAIR_MAX_TERMS) return SPK_ERR_ARG;
        if (!p->a_pow || !p->a_div || !p->coefficients || !p->exponents) return SPK_ERR_ARG;
    }
    if (p->kind == SPK_PAIR_DAMPED_COULOMB && !(p->switch_off != p->switch_on)) return SPK_ERR_ARG;
    if (p->kind == SPK_PAIR_EWALD_REAL && !(p->alpha > 0.0)) return SPK_ERR_ARG;
    return SPK_OK;
}

}  // namespace

#define GRID1D(n, T) (unsigned)spk_cdiv((n), (T)), (T), 0, spk_st(stream)

extern "C" size_t spk_pair_energy_workspace_bytes(int64_t n_edges, int64_t n_sys) {
    const int64_t nb = n_edges > 0 ? spk_cdiv(n_edges, PE_T) : 0;
    return sizeof(double) * (size_t)((n_sys > 0 ? n_sys : 0) + nb + 1);
}

extern "C" int spk_pair_energy_fwd(const spk_pair_t* p, const float* r_ij, const int64_t* idx_i, const int64_t* idx_j,
                                   const int64_t* Z, const float* q, const int64_t* idx_m, const int32_t* rowptr,
                                   const int32_t* slot_eid, const int32_t* sys_ptr, int64_t n_edges, int64_t n_sys,
                                   float* energy, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (n_edges < 0 || n_sys < 0 || n_edges >= (1ll << 31) - 1) return SPK_ERR_ARG;
    const int rc = check_pair(p);
    if (rc != SPK_OK) return rc;
    if (n_sys == 0) return SPK_OK;
    if (!rowptr || !sys_ptr || !energy || !workspace) return SPK_ERR_ARG;
    if (workspace_bytes < spk_pair_energy_workspace_bytes(n_edges, n_sys)) return SPK_ERR_ARG;
    if (n_edges > 0 && (!r_ij || !idx_i || !idx_j || !idx_m || !slot_eid)) return SPK_ERR_ARG;
    if (n_edges > 0 && (p->kind == SPK_PAIR_ZBL ? !Z : !q)) return SPK_ERR_ARG;
    double* sys_part = reinterpret_cast<double*>(workspace);
    double* head = sys_part + n_sys;
    const cudaStream_t st = spk_st(stream);
    if (n_edges > 0)
        spk_launch(k_pair_partials, (unsigned)spk_cdiv(n_edges, PE_T), PE_T, 0, st, *p, r_ij, idx_i, idx_j, Z, q, idx_m,
                   rowptr, slot_eid, sys_ptr, n_sys, sys_part, head);
    spk_launch(k_pair_finish, (unsigned)n_sys, SEG_FIN_T, 0, st, rowptr, sys_ptr, sys_part, head, 0.5 * p->ke, energy);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_pair_energy_bwd(const spk_pair_t* p, const float* r_ij, const int64_t* idx_i, const int64_t* idx_j,
                                   const int64_t* Z, const float* q, const int64_t* idx_m, const float* g_E,
                                   const int32_t* rowptr, const int32_t* slot_j, const int32_t* slot_eid,
                                   const int32_t* sptr, const int32_t* pos_slot, const int32_t* pos_i, int64_t n_atoms,
                                   int64_t n_edges, float* g_rij, float* g_q, spk_stream_t stream) {
    if (n_edges < 0 || n_atoms < 0 || n_edges >= (1ll << 31) - 1) return SPK_ERR_ARG;
    const int rc = check_pair(p);
    if (rc != SPK_OK) return rc;
    const bool coul = p->kind != SPK_PAIR_ZBL;
    if (n_edges > 0 && (!r_ij || !idx_i || !idx_j || !idx_m || !g_E || !g_rij || (coul ? !q : !Z))) return SPK_ERR_ARG;
    if (g_q && (!coul || !q || !idx_m || !g_E || !rowptr || !slot_j || !slot_eid || !sptr || !pos_slot || !pos_i))
        return SPK_ERR_ARG;
    const double scale = 0.5 * p->ke;
    if (n_edges > 0)
        spk_launch(k_pair_grad_rij, GRID1D(n_edges, 256), *p, r_ij, idx_i, idx_j, Z, q, idx_m, g_E, n_edges, scale, g_rij);
    if (g_q && n_atoms > 0)
        spk_launch(k_pair_grad_q, GRID1D(n_atoms, 128), *p, r_ij, q, idx_m, g_E, rowptr, slot_j, slot_eid, sptr, pos_slot,
                   pos_i, n_atoms, scale, g_q);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

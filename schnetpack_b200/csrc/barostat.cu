// Nose-Hoover-chain barostats of the device-resident MD step (md/simulation_hooks/barostats.py:162-927, with the position /
// momentum propagation that md/integrators.py:232-263 NPTVelocityVerlet delegates to them), isotropic and anisotropic, for
// one chain per system or one per degree of freedom (massive).  Every entry point only enqueues work, so a whole NPT step
// can be captured into one CUDA graph.
//
// Per-system sums (kinetic energy and kinetic-energy tensor) use the fixed-shape segmented reduction of segscan.cuh: CTAs
// of KT consecutive atoms write one fp64 partial per (system, CTA) pair, one CTA per system adds them in a fixed order.  No
// atomics touch a sum.  The per-system work (chains, barostat force, the 3x3 operators with their Jacobi eigendecomposition) runs
// one thread per system; the per-atom kernels apply the resulting operators.
#include "md_common.cuh"

namespace {

constexpr int KT = 256;   // atoms per CTA of the partial pass
constexpr int NK = 7;     // |p|^2/m, then p_x p_x, p_y p_y, p_z p_z, p_x p_y, p_x p_z, p_y p_z (all / m)
constexpr int ELT_T = 256;

struct Workspace {
    double* sys_part;  // [n_sys, NK]
    double* scale;     // [n_sys]
    double* ops;       // [n_sys, 18]: operator A, operator B (row-major 3x3 each)
    double* tot;       // [n_sys, NK]: per-system totals of the partials
    double* head;      // [n_blocks, NK]
};

static inline int64_t k_blocks(int64_t n_atoms) { return spk_cdiv(n_atoms, KT); }

static inline Workspace carve(void* ws, int64_t n_sys) {
    double* d = reinterpret_cast<double*>(ws);
    return Workspace{d, d + NK * n_sys, d + (NK + 1) * n_sys, d + (NK + 19) * n_sys, d + (2 * NK + 19) * n_sys};
}

__global__ void __launch_bounds__(KT) k_ke7_partials(const float* __restrict__ p, const float* __restrict__ m,
                                                     const int64_t* __restrict__ idx_m, const int32_t* __restrict__ sys_ptr,
                                                     int64_t n_atoms, double* __restrict__ sys_part,
                                                     double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * KT + threadIdx.x;
    double v[NK];
#pragma unroll
    for (int c = 0; c < NK; ++c) v[c] = 0.0;
    int64_t s = 0, first = 0, end = 0;
    if (a < n_atoms) {
        const double px = p[3 * a], py = p[3 * a + 1], pz = p[3 * a + 2], ma = (double)m[a];
        v[0] = (px * px + py * py + pz * pz) / ma;             // system.py:383-385
        v[1] = px * px / ma;                                   // system.py:399-403
        v[2] = py * py / ma;
        v[3] = pz * pz / ma;
        v[4] = px * py / ma;
        v[5] = px * pz / ma;
        v[6] = py * pz / ma;
        s = idx_m[a];
        first = sys_ptr[s];
        end = sys_ptr[s + 1];
    }
    seg_partials<KT, NK>(v, n_atoms, s, first, end, sys_part, head);
}

// 2 KE (= sum |p|^2/m) and 2 K (= sum p p^T / m, row-major 3x3) of system s
__device__ __forceinline__ void system_ke(const int32_t* __restrict__ sys_ptr, const Workspace& w, int64_t s,
                                          double& ke2, double (&k2)[9]) {
    const double* acc = w.tot + s * NK;
    ke2 = acc[0];
    k2[0] = acc[1]; k2[4] = acc[2]; k2[8] = acc[3];
    k2[1] = k2[3] = acc[4];
    k2[2] = k2[6] = acc[5];
    k2[5] = k2[7] = acc[6];
}

__device__ __forceinline__ spk_nhc_params_t chain_params(const spk_nhc_barostat_t& b) {
    spk_nhc_params_t q;
    q.chain_length = b.chain_length;
    q.multi_step = b.multi_step;
    q.order = b.order;
    q.massive = b.massive;
    q.kb_temperature = b.kb_temperature;
    for (int k = 0; k < 7; ++k) q.time_step[k] = b.ys_time_step[k];
    return q;
}

// barostats.py:408-481 (_update_thermostat), one thread per system: the particle chain (unless massive) and the cell chain
__global__ void k_baro_thermostat(const __grid_constant__ spk_nhc_barostat_t b, const int32_t* __restrict__ sys_ptr,
                                  int64_t n_sys, Workspace w) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_sys) return;
    const spk_nhc_params_t q = chain_params(b);
    const int L = b.chain_length;
    if (!b.massive) {
        double ke2, k2[9];
        system_ke(sys_ptr, w, s, ke2, k2);
        const double dof = 3.0 * (double)(sys_ptr[s + 1] - sys_ptr[s]);
        w.scale[s] = nhc_propagate(ke2, dof, q, q.kb_temperature, b.t_v + s * L, b.t_f + s * L, b.t_m + s * L);
    }
    const int nb = b.anisotropic ? 9 : 1;
    double* bv = b.b_v + s * nb;
    double ke_cell = 0.0;                           // :501-508, :810-820
    if (b.anisotropic) {
        double sq = 0.0;
        for (int k = 0; k < 9; ++k) sq += bv[k] * bv[k];
        ke_cell = b.b_m[s] * sq;
    } else {
        ke_cell = b.b_m[s] * (bv[0] * bv[0]);
    }
    const double sc = nhc_propagate(ke_cell, b.anisotropic ? 6.0 : 1.0, q, q.kb_temperature, b.c_v + s * L, b.c_f + s * L,
                                    b.c_m + s * L);
    for (int k = 0; k < nb; ++k) bv[k] = bv[k] * sc;          // :473-481, :798-808
}

// barostats.py:604-631 / :822-842 (_update_barostat): barostat force from the pressure, then b_v += 1/2 dt b_f.
// stress = virial_scale * virial / V with V the volume of the MD cell.
__global__ void k_baro_kick(const __grid_constant__ spk_nhc_barostat_t b, const int32_t* __restrict__ sys_ptr,
                            int64_t n_sys, const double* __restrict__ cell, const double* __restrict__ virial,
                            double virial_scale, Workspace w) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_sys) return;
    double ke2, k2[9];
    system_ke(sys_ptr, w, s, ke2, k2);
    const double dof = 3.0 * (double)(sys_ptr[s + 1] - sys_ptr[s]);
    const double V = det3(cell + s * 9);
    double stress[9];
    for (int k = 0; k < 9; ++k) stress[k] = virial_scale * virial[s * 9 + k] / V;
    const double P0 = b.target_pressure, bm = b.b_m[s];
    if (b.anisotropic) {
        for (int k = 0; k < 9; ++k) {
            const bool diag = (k % 4) == 0;
            const double pt = -stress[k] + k2[k] / V;                              // system.py:604-608
            const double bf = (V * (pt - (diag ? P0 : 0.0)) + (diag ? ke2 / dof : 0.0)) / bm;
            b.b_f[s * 9 + k] = bf;
            b.b_v[s * 9 + k] = b.b_v[s * 9 + k] + 0.5 * b.time_step * bf;
        }
    } else {
        const double P = ((-stress[0]) + (-stress[4]) + (-stress[8])) / 3.0;       // system.py:609-610
        const double bf = ((1.0 + 3.0 / dof) * ke2 + 3.0 * V * (P - P0)) / bm;
        b.b_f[s] = bf;
        b.b_v[s] = b.b_v[s] + 0.5 * b.time_step * bf;
    }
}

// The per-system operators of propagate_half_step (main = 0, :661-686 / :885-926) and propagate_main_step (main = 1,
// :633-659 / :844-883): x' = x A + c y B per atom (row vectors).  The main step also scales the MD cell and writes the model
// cell (= MD cell * position_conversion).
__global__ void k_baro_operators(const __grid_constant__ spk_nhc_barostat_t b, const int32_t* __restrict__ sys_ptr,
                                 int64_t n_sys, int main_step, double* __restrict__ cell, float* __restrict__ model_cell,
                                 double position_conversion, Workspace w) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_sys) return;
    const double dt = b.time_step;
    const double dof = 3.0 * (double)(sys_ptr[s + 1] - sys_ptr[s]);
    double* A = w.ops + s * 18;
    double* B = A + 9;
    double* c = main_step ? cell + s * 9 : nullptr;
    if (!b.anisotropic) {
        const double bv = b.b_v[s];
        double a, bb;
        if (main_step) {
            const double x = dt * bv;
            a = exp(0.5 * x);
            bb = a * stable_sinh_div(0.5 * x);
            const double cc = exp(x);
            for (int k = 0; k < 9; ++k) c[k] = c[k] * cc;
        } else {
            const double x = 0.25 * dt * bv * (1.0 + 3.0 / dof);
            a = exp(-x);
            bb = a * stable_sinh_div(x);
        }
        for (int k = 0; k < 9; ++k) {
            A[k] = (k % 4) == 0 ? a * a : 0.0;
            B[k] = (k % 4) == 0 ? bb : 0.0;
        }
    } else {
        double lam[3], Q[3][3];
        sym3_eig(b.b_v + s * 9, lam, Q);
        double da[3], db[3];
        if (main_step) {
            for (int k = 0; k < 3; ++k) {
                const double x = lam[k] * dt;
                const double ca = exp(0.5 * x);
                da[k] = ca * ca;
                db[k] = ca * stable_sinh_div(0.5 * x);
            }
        } else {
            const double tr = lam[0] + lam[1] + lam[2];
            for (int k = 0; k < 3; ++k) {
                const double x = (lam[k] + tr / dof) * dt * 0.5;
                const double ca = exp(-0.5 * x);
                da[k] = ca * ca;
                db[k] = ca * stable_sinh_div(0.5 * x);
            }
        }
        sym3_compose(Q, da, A);
        sym3_compose(Q, db, B);
        if (main_step) {                                        // cells @ operator_a
            double n[9];
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) n[i * 3 + j] = c[i * 3] * A[j] + c[i * 3 + 1] * A[3 + j] + c[i * 3 + 2] * A[6 + j];
            for (int k = 0; k < 9; ++k) c[k] = n[k];
        }
    }
    if (main_step && model_cell)
        for (int k = 0; k < 9; ++k) model_cell[s * 9 + k] = (float)(c[k] * position_conversion);
}

// x[a] = x[a] A_s + c y[a] B_s / (m[a] if given), s = system of atom a; also model_x = x * position_conversion if given
__global__ void k_baro_apply(float* __restrict__ x, float* __restrict__ model_x, const float* __restrict__ y,
                             const float* __restrict__ m, const int64_t* __restrict__ idx_m, int64_t n_atoms, double coef,
                             float position_conversion, Workspace w) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const double* A = w.ops + idx_m[a] * 18;
    const double* B = A + 9;
    const double inv = m ? 1.0 / (double)m[a] : 1.0;
    const double x0 = x[3 * a], x1 = x[3 * a + 1], x2 = x[3 * a + 2];
    const double y0 = y[3 * a] * inv, y1 = y[3 * a + 1] * inv, y2 = y[3 * a + 2] * inv;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const double ux = x0 * A[j] + x1 * A[3 + j] + x2 * A[6 + j];
        const double uy = y0 * B[j] + y1 * B[3 + j] + y2 * B[6 + j];
        const float v = (float)(ux + coef * uy);
        x[3 * a + j] = v;
        if (model_x) model_x[3 * a + j] = v * position_conversion;
    }
}

static bool params_ok(const spk_nhc_barostat_t* b) {
    return b && b->chain_length >= 1 && b->multi_step >= 1 && (b->order == 3 || b->order == 5 || b->order == 7) &&
           b->kb_temperature > 0.0 && b->t_v && b->t_f && b->t_m && b->c_v && b->c_f && b->c_m && b->b_v && b->b_f &&
           b->b_m;
}

static int check(const spk_nhc_barostat_t* b, const float* momenta, const float* masses, const int64_t* idx_m,
                 const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, void* workspace, size_t workspace_bytes) {
    if (!params_ok(b)) return SPK_ERR_ARG;
    if (n_atoms < 0 || n_sys <= 0 || n_atoms >= (1ll << 31) / 3) return SPK_ERR_ARG;
    if (!sys_ptr || !workspace || workspace_bytes < spk_md_barostat_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!momenta || !masses || !idx_m)) return SPK_ERR_ARG;
    return SPK_OK;
}

// per-system sums of the NK kinetic terms into w.tot: CTA partials, then the fixed-order per-system pass
static void ke_partials(const float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                        int64_t n_atoms, int64_t n_sys, const Workspace& w, cudaStream_t st) {
    if (n_atoms > 0)
        spk_launch(k_ke7_partials, (unsigned)k_blocks(n_atoms), KT, 0, st, momenta, masses, idx_m, sys_ptr, n_atoms,
                   w.sys_part, w.head);
    spk_launch(k_seg_finish<KT, NK>, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, (const int32_t*)nullptr, w.sys_part,
               w.head, w.tot);
}

__global__ void k_ke_tensor_system(const int32_t* __restrict__ sys_ptr, int64_t n_sys, Workspace w, double* __restrict__ out) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_sys) return;
    double ke2, k2[9];
    system_ke(sys_ptr, w, s, ke2, k2);
    for (int k = 0; k < 9; ++k) out[s * 9 + k] = 0.5 * k2[k];
}

#define SYS_GRID(n) (unsigned)spk_cdiv((n), 128), 128, 0, st

}  // namespace

extern "C" size_t spk_md_barostat_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? k_blocks(n_atoms) : 0;
    return sizeof(double) * (size_t)((2 * NK + 19) * (n_sys > 0 ? n_sys : 0) + NK * nb + 1);
}

extern "C" int spk_md_kinetic_energy_tensor(const float* momenta, const float* masses, const int64_t* idx_m,
                                            const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, double* ke_tensor,
                                            void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (n_atoms < 0 || n_sys <= 0 || n_atoms >= (1ll << 31) - 1 || !ke_tensor || !sys_ptr || !workspace) return SPK_ERR_ARG;
    if (workspace_bytes < spk_md_barostat_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!momenta || !masses || !idx_m)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    const Workspace w = carve(workspace, n_sys);
    ke_partials(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, w, st);
    spk_launch(k_ke_tensor_system, SYS_GRID(n_sys), sys_ptr, n_sys, w, ke_tensor);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_barostat_thermostat(const spk_nhc_barostat_t* b, float* momenta, const float* masses,
                                          const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys,
                                          void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    const int rc = check(b, momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes);
    if (rc != SPK_OK) return rc;
    cudaStream_t st = spk_st(stream);
    const Workspace w = carve(workspace, n_sys);
    if (!b->massive) ke_partials(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, w, st);
    spk_launch(k_baro_thermostat, SYS_GRID(n_sys), *b, sys_ptr, n_sys, w);
    if (n_atoms > 0) {
        if (b->massive) {
            spk_nhc_params_t q = {b->chain_length, b->multi_step, b->order, 1, b->kb_temperature, {}};
            for (int k = 0; k < 7; ++k) q.time_step[k] = b->ys_time_step[k];
            spk_launch(k_nhc_massive, (unsigned)spk_cdiv(n_atoms * 3, 128), 128, 0, st, momenta, masses, n_atoms * 3, q,
                       nullptr, nullptr, b->t_v, b->t_f, b->t_m);
        } else {
            spk_launch(k_scale_momenta, (unsigned)spk_cdiv(n_atoms * 3, ELT_T), ELT_T, 0, st, momenta, idx_m, w.scale,
                       n_atoms * 3);
        }
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_barostat_kick(const spk_nhc_barostat_t* b, const float* momenta, const float* masses,
                                    const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys,
                                    const double* cell, const double* virial, double virial_scale, void* workspace,
                                    size_t workspace_bytes, spk_stream_t stream) {
    const int rc = check(b, momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes);
    if (rc != SPK_OK) return rc;
    if (!cell || !virial) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    const Workspace w = carve(workspace, n_sys);
    ke_partials(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, w, st);
    spk_launch(k_baro_kick, SYS_GRID(n_sys), *b, sys_ptr, n_sys, cell, virial, virial_scale, w);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_barostat_half_step(const spk_nhc_barostat_t* b, float* momenta, const float* forces,
                                         double force_conversion, const int64_t* idx_m, const int32_t* sys_ptr,
                                         int64_t n_atoms, int64_t n_sys, void* workspace, size_t workspace_bytes,
                                         spk_stream_t stream) {
    const int rc = check(b, momenta, forces, idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes);
    if (rc != SPK_OK) return rc;
    cudaStream_t st = spk_st(stream);
    const Workspace w = carve(workspace, n_sys);
    spk_launch(k_baro_operators, SYS_GRID(n_sys), *b, sys_ptr, n_sys, 0, (double*)nullptr, (float*)nullptr, 1.0, w);
    if (n_atoms > 0)
        spk_launch(k_baro_apply, (unsigned)spk_cdiv(n_atoms, ELT_T), ELT_T, 0, st, momenta, (float*)nullptr, forces,
                   (const float*)nullptr, idx_m, n_atoms, 0.5 * b->time_step * force_conversion, 1.0f, w);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_barostat_main_step(const spk_nhc_barostat_t* b, float* positions, float* model_positions,
                                         const float* momenta, const float* masses, const int64_t* idx_m,
                                         const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, double* cell,
                                         float* model_cell, double position_conversion, void* workspace,
                                         size_t workspace_bytes, spk_stream_t stream) {
    const int rc = check(b, momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes);
    if (rc != SPK_OK) return rc;
    if (!cell || (n_atoms > 0 && !positions)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    const Workspace w = carve(workspace, n_sys);
    spk_launch(k_baro_operators, SYS_GRID(n_sys), *b, sys_ptr, n_sys, 1, cell, model_cell, position_conversion, w);
    if (n_atoms > 0)
        spk_launch(k_baro_apply, (unsigned)spk_cdiv(n_atoms, ELT_T), ELT_T, 0, st, positions, model_positions, momenta,
                   masses, idx_m, n_atoms, b->time_step, (float)position_conversion, w);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

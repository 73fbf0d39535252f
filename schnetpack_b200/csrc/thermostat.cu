// Thermostats of the device-resident MD step (md/simulation_hooks/thermostats.py:149-513): per-system kinetic energies,
// Berendsen rescaling, Nose-Hoover-chain propagation (per system or massive) and the Langevin kick with a counter-based
// Philox4x32-10 generator.  Every entry point only enqueues work, so a whole NVT step can be captured into one CUDA graph.
//
// Per-system sums are deterministic: the atoms are cut into CTAs of KE_T consecutive atoms, and the partial pass of
// segscan.cuh leaves one fp64 partial per (system, CTA) pair.  k_thermo_system then adds a system's partials in CTA order,
// one thread per system.  No atomics touch a sum, so the result is bitwise the same on every call, whatever the size mix of
// the batch (one 262 144-atom box spans 1024 CTAs, a 1-atom system one).
#include "md_common.cuh"

namespace {

constexpr int KE_T = 256;  // atoms per CTA of the partial pass
constexpr int ELT_T = 256;

enum ThermoMode { MODE_KE = 0, MODE_BERENDSEN = 1, MODE_NHC = 2 };

struct Workspace {
    double* sys_part;  // [n_sys]
    double* scale;     // [n_sys]
    double* head;      // [n_blocks]
};

static inline int64_t ke_blocks(int64_t n_atoms) { return spk_cdiv(n_atoms, KE_T); }

static inline Workspace carve(void* ws, int64_t n_sys) {
    double* d = reinterpret_cast<double*>(ws);
    return Workspace{d, d + n_sys, d + 2 * n_sys};
}

__global__ void __launch_bounds__(KE_T) k_ke_partials(const float* __restrict__ p, const float* __restrict__ m,
                                                      const int64_t* __restrict__ idx_m,
                                                      const int32_t* __restrict__ sys_ptr, int64_t n_atoms,
                                                      double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * KE_T + threadIdx.x;
    double v[1] = {0.0};
    int64_t s = 0, first = 0, end = 0;
    if (a < n_atoms) {
        const double px = p[3 * a], py = p[3 * a + 1], pz = p[3 * a + 2];
        v[0] = (px * px + py * py + pz * pz) / (double)m[a];
        s = idx_m[a];
        first = sys_ptr[s];
        end = sys_ptr[s + 1];
    }
    seg_partials<KE_T, 1>(v, n_atoms, s, first, end, sys_part, head);
}

// sum_{a in s} p_a^2 / m_a in CTA order (0 for an empty system)
__device__ __forceinline__ double system_sum(const int32_t* __restrict__ sys_ptr, const double* __restrict__ sys_part,
                                             const double* __restrict__ head, int64_t s) {
    const int64_t a0 = sys_ptr[s], a1 = sys_ptr[s + 1];
    if (a1 <= a0) return 0.0;
    double acc = sys_part[s];
    for (int64_t b = a0 / KE_T + 1; b <= (a1 - 1) / KE_T; ++b) acc += head[b];
    return acc;
}

// one thread per system: finish the sum, then the temperature (system.py:407-421) and the mode's scaling factor.  NHC
// chains use kbt_sys[s] (nullable: q.kb_temperature for every system).
__global__ void k_thermo_system(const int32_t* __restrict__ sys_ptr, int64_t n_sys, const double* __restrict__ sys_part,
                                const double* __restrict__ head, int mode, double kB, double dt_over_tau, double t_bath,
                                const __grid_constant__ spk_nhc_params_t q, const double* __restrict__ kbt_sys,
                                double* __restrict__ chain_v,
                                double* __restrict__ chain_f, const double* __restrict__ chain_m, double* __restrict__ ke_out,
                                double* __restrict__ temp_out, double* __restrict__ scale) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_sys) return;
    const double sum = system_sum(sys_ptr, sys_part, head, s);
    const double n = (double)(sys_ptr[s + 1] - sys_ptr[s]);
    const double ke = 0.5 * sum;
    const double temp = n > 0.0 ? 2.0 / (3.0 * n * kB) * ke : 0.0;
    if (mode == MODE_KE) {
        if (ke_out) ke_out[s] = ke;
        if (temp_out) temp_out[s] = temp;
        return;
    }
    double sc = 1.0;
    if (mode == MODE_BERENDSEN) {
        // thermostats.py:181-186; a system at rest has nothing to rescale
        if (temp > 0.0) sc = sqrt(1.0 + dt_over_tau * (t_bath / temp - 1.0));
    } else {
        const int L = q.chain_length;
        const double kbt = kbt_sys ? kbt_sys[s] : q.kb_temperature;
        sc = nhc_propagate(2.0 * ke, 3.0 * n, q, kbt, chain_v + s * L, chain_f + s * L, chain_m + s * L);   // :489
    }
    scale[s] = sc;
}

// thermostats.py:244-261: p = c1 p + sqrt(m kB T) c2 xi, one thread per atom (xi = the first three normals of its draw).
// kB T is kbt, or kbt_sys[idx_m[a]] when the per-system table is given.  counter: the application index and its ticket
// (advance_counter).
__global__ void k_langevin(float* __restrict__ p, const float* __restrict__ m, const int64_t* __restrict__ idx_m,
                           int64_t n_atoms, double c1, double c2, double kbt, const double* __restrict__ kbt_sys,
                           uint64_t seed, unsigned long long* counter) {
    SPK_PDL_ENTER();
    const unsigned long long app = *(volatile unsigned long long*)counter;
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a < n_atoms) {
        const uint4 x = philox_draw(seed, app, a);
        const double2 z01 = box_muller(x.x, x.y), z23 = box_muller(x.z, x.w);
        const double fac = sqrt((double)m[a] * (kbt_sys ? kbt_sys[idx_m[a]] : kbt)) * c2;
        p[3 * a + 0] = (float)(c1 * (double)p[3 * a + 0] + fac * z01.x);
        p[3 * a + 1] = (float)(c1 * (double)p[3 * a + 1] + fac * z01.y);
        p[3 * a + 2] = (float)(c1 * (double)p[3 * a + 2] + fac * z23.x);
    }
    advance_counter(counter, app);
}

__global__ void k_philox_bits(uint64_t seed, const unsigned long long* __restrict__ counter, int64_t n,
                              uint4* __restrict__ out) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) out[i] = philox_draw(seed, counter[0], i);
}

static int check_systems(const float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                         int64_t n_atoms, int64_t n_sys, void* workspace, size_t workspace_bytes) {
    if (n_atoms < 0 || n_sys <= 0 || n_atoms >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (!sys_ptr || !workspace || workspace_bytes < spk_md_thermostat_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!momenta || !masses || !idx_m)) return SPK_ERR_ARG;
    return SPK_OK;
}

static int thermo_systems(int mode, float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                          int64_t n_atoms, int64_t n_sys, double kB, double dt_over_tau, double t_bath,
                          const spk_nhc_params_t* q, const double* kbt_sys, double* chain_v, double* chain_f,
                          const double* chain_m, double* ke, double* temperature, void* workspace, size_t workspace_bytes,
                          spk_stream_t stream) {
    const int rc = check_systems(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes);
    if (rc != SPK_OK) return rc;
    cudaStream_t st = spk_st(stream);
    Workspace w = carve(workspace, n_sys);
    spk_nhc_params_t qq = {};
    if (q) qq = *q;
    if (n_atoms > 0)
        spk_launch(k_ke_partials, (unsigned)ke_blocks(n_atoms), KE_T, 0, st, momenta, masses, idx_m, sys_ptr, n_atoms,
                   w.sys_part, w.head);
    spk_launch(k_thermo_system, (unsigned)spk_cdiv(n_sys, 128), 128, 0, st, sys_ptr, n_sys, w.sys_part, w.head, mode, kB,
               dt_over_tau, t_bath, qq, kbt_sys, chain_v, chain_f, chain_m, ke, temperature, w.scale);
    if (mode != MODE_KE && n_atoms > 0)
        spk_launch(k_scale_momenta, (unsigned)spk_cdiv(n_atoms * 3, ELT_T), ELT_T, 0, st, momenta, idx_m, w.scale,
                   n_atoms * 3);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

// params->kb_temperature is checked only when no per-system table replaces it
static bool nhc_params_ok(const spk_nhc_params_t* q, bool per_system) {
    return q && q->chain_length >= 1 && q->multi_step >= 1 && (q->order == 3 || q->order == 5 || q->order == 7) &&
           (per_system || q->kb_temperature > 0.0);
}

static int nhc(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
               int64_t n_sys, const spk_nhc_params_t* params, const double* kbt_sys, double* chain_v, double* chain_f,
               const double* chain_m, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (!nhc_params_ok(params, kbt_sys != nullptr) || !chain_v || !chain_f || !chain_m) return SPK_ERR_ARG;
    if (params->massive) {
        if (n_atoms < 0 || n_atoms >= (1ll << 31) / 3) return SPK_ERR_ARG;
        if (n_atoms == 0) return SPK_OK;
        if (!momenta || !masses || (kbt_sys && !idx_m)) return SPK_ERR_ARG;
        spk_launch(k_nhc_massive, (unsigned)spk_cdiv(n_atoms * 3, 128), 128, 0, spk_st(stream), momenta, masses,
                   n_atoms * 3, *params, idx_m, kbt_sys, chain_v, chain_f, chain_m);
        SPK_LAUNCH_CHECK();
        return SPK_OK;
    }
    return thermo_systems(MODE_NHC, momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, 1.0, 0.0, 0.0, params, kbt_sys,
                          chain_v, chain_f, chain_m, nullptr, nullptr, workspace, workspace_bytes, stream);
}

static int langevin(float* momenta, const float* masses, const int64_t* idx_m, int64_t n_atoms, double c1, double c2,
                    double kb_temperature, const double* kbt_sys, uint64_t seed, uint64_t* counter, spk_stream_t stream) {
    if (n_atoms < 0 || n_atoms >= (1ll << 31) - 1 || !counter || !(kb_temperature >= 0.0)) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!momenta || !masses || (kbt_sys && !idx_m)) return SPK_ERR_ARG;
    spk_launch(k_langevin, (unsigned)spk_cdiv(n_atoms, ELT_T), ELT_T, 0, spk_st(stream), momenta, masses, idx_m, n_atoms,
               c1, c2, kb_temperature, kbt_sys, seed, reinterpret_cast<unsigned long long*>(counter));
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

}  // namespace

extern "C" size_t spk_md_thermostat_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? ke_blocks(n_atoms) : 0;
    return sizeof(double) * (size_t)(2 * (n_sys > 0 ? n_sys : 0) + nb + 1);
}

extern "C" int spk_md_kinetic_energy(const float* momenta, const float* masses, const int64_t* idx_m,
                                     const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, double kB, double* ke,
                                     double* temperature, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (!(kB > 0.0) || (!ke && !temperature)) return SPK_ERR_ARG;
    return thermo_systems(MODE_KE, const_cast<float*>(momenta), masses, idx_m, sys_ptr, n_atoms, n_sys, kB, 0.0, 0.0,
                          nullptr, nullptr, nullptr, nullptr, nullptr, ke, temperature, workspace, workspace_bytes, stream);
}

extern "C" int spk_md_berendsen(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                                int64_t n_atoms, int64_t n_sys, double kB, double dt_over_tau, double temperature_bath,
                                void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (!(kB > 0.0) || !(dt_over_tau >= 0.0) || !(temperature_bath >= 0.0)) return SPK_ERR_ARG;
    return thermo_systems(MODE_BERENDSEN, momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, kB, dt_over_tau,
                          temperature_bath, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, workspace,
                          workspace_bytes, stream);
}

extern "C" int spk_md_nhc(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                          int64_t n_atoms, int64_t n_sys, const spk_nhc_params_t* params, double* chain_v,
                          double* chain_f, const double* chain_m, void* workspace, size_t workspace_bytes,
                          spk_stream_t stream) {
    return nhc(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, params, nullptr, chain_v, chain_f, chain_m, workspace,
               workspace_bytes, stream);
}

extern "C" int spk_md_nhc_per_system(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                                     int64_t n_atoms, int64_t n_sys, const spk_nhc_params_t* params,
                                     const double* kb_temperature_sys, double* chain_v, double* chain_f,
                                     const double* chain_m, void* workspace, size_t workspace_bytes,
                                     spk_stream_t stream) {
    if (!kb_temperature_sys) return SPK_ERR_ARG;
    return nhc(momenta, masses, idx_m, sys_ptr, n_atoms, n_sys, params, kb_temperature_sys, chain_v, chain_f, chain_m,
               workspace, workspace_bytes, stream);
}

extern "C" int spk_md_langevin(float* momenta, const float* masses, int64_t n_atoms, double c1, double c2,
                               double kb_temperature, uint64_t seed, uint64_t* counter, spk_stream_t stream) {
    return langevin(momenta, masses, nullptr, n_atoms, c1, c2, kb_temperature, nullptr, seed, counter, stream);
}

extern "C" int spk_md_langevin_per_system(float* momenta, const float* masses, const int64_t* idx_m, int64_t n_atoms,
                                          double c1, double c2, const double* kb_temperature_sys, uint64_t seed,
                                          uint64_t* counter, spk_stream_t stream) {
    if (!kb_temperature_sys) return SPK_ERR_ARG;
    return langevin(momenta, masses, idx_m, n_atoms, c1, c2, 0.0, kb_temperature_sys, seed, counter, stream);
}

extern "C" int spk_philox4x32_10(uint64_t seed, const uint64_t* counter, int64_t n, uint32_t* out, spk_stream_t stream) {
    if (n < 0 || !counter || (n > 0 && !out)) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    spk_launch(k_philox_bits, (unsigned)spk_cdiv(n, ELT_T), ELT_T, 0, spk_st(stream), seed,
               reinterpret_cast<const unsigned long long*>(counter), n, reinterpret_cast<uint4*>(out));
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

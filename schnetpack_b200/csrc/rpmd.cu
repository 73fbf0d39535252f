// Ring-polymer MD of the device MD step: the normal-mode transform (md/utils/normal_model_transformation.py:37-101), the
// free ring-polymer propagation of the RingPolymer integrator (md/integrators.py:154-229) and the ring-polymer thermostats
// PILE-L / PILE-G / TRPMD and NHC (md/simulation_hooks/thermostats_rpmd.py:33-234,373-501), and the PILE barostat of
// ring-polymer NPT (md/simulation_hooks/barostats_rpmd.py:21-208 with md/integrators.py:266-305 NPTRingPolymer), and the
// colored-noise GLE / RPMD-GLE / PIGLET thermostats (md/simulation_hooks/thermostats.py:527-730, thermostats_rpmd.py:
// 237-370; the classical GLE runs as P = 1 with C = [[1]]).  Every entry point only enqueues work, so the whole RPMD step
// stays one CUDA graph.
//
// Bead arrays are [P, n_atoms, 3] fp32, replica-major, so for a fixed bead a run of consecutive degrees of freedom (atom,
// component) is contiguous.  The mode kernels give a CTA RP_T = 32 consecutive degrees of freedom across all P beads: the
// bead values are staged in shared memory with coalesced loads, every (mode, dof) pair is formed as an fp64 dot product with
// a row of C, the per-mode operator is applied in registers, and the back-transform C^T writes the beads.  Threads of a warp
// share one mode (or bead) index, so their reads of C are warp-uniform broadcasts from L1.  Shared memory: 24 P RP_T bytes,
// 48 KB at P = 64.
//
// The per-system centroid sums of the global thermostats use the fixed-shape segmented scan of segscan.cuh and one ordered
// finishing pass per system: no atomics touch a sum, so every call is bitwise reproducible.  The barostat's half step
// forms its three per-system sums over the mode-0 forces and momenta the same way; its finishing CTA also averages the
// P bead volumes and virials of its system and updates the cell momentum.
#include "md_common.cuh"

namespace {

constexpr int RP_T = 32;          // degrees of freedom per CTA of the mode kernels
constexpr int RP_THREADS = 256;
constexpr int RP_KT = 256;        // atoms per CTA of the centroid partial pass
constexpr int RP_NV = 2;          // centroid sums: sum |p~_0|^2 / m, sum |xi_0|^2
constexpr int RP_MAX_BEADS = 64;
constexpr int RB_NV = 3;          // barostat sums: sum F~_0 . p~_0 / m, sum |F~_0|^2 / (3 m), sum |p_bar|^2 / m
constexpr int GLE_MAX_D = 16;     // extended momenta per degree of freedom (p~ plus up to 15 auxiliary momenta)

enum RpmdOp { OP_MAIN = 0, OP_PILE = 1, OP_NHC = 2, OP_BARO = 3, OP_GLE = 4 };

struct RpmdArgs {
    float* x;                     // bead positions (OP_MAIN)
    float* p;                     // bead momenta
    float* model_x;               // nullable: x * pos_conv (OP_MAIN)
    const float* m;               // [n_atoms]
    const int64_t* idx_m;
    const int32_t* sys_ptr;
    const double* C;              // [P, P]
    const double* prop;           // [P, 2, 2] (OP_MAIN, OP_BARO)
    const double* baro_ab;        // [n_sys, 2] per-system (a, b) of the barostat's centroid propagation (OP_BARO)
    const double* c1;             // [P] (OP_PILE)
    const double* c2;
    const double* tot;            // [n_sys, RP_NV] centroid sums (global variants)
    double* chain_v;              // [P * 3 n_atoms, L] (OP_NHC)
    double* chain_f;
    const double* chain_m;
    unsigned long long* counter;  // [2]: application index, ticket (OP_PILE, OP_GLE)
    double* gle_s;                // [P * 3 n_atoms, D] extended momenta, row k 3 n_atoms + i (OP_GLE)
    const double* gle_c1;         // [n_mats, D, D] drift propagator exp(-dt/2 A), row-major (OP_GLE)
    const double* gle_c2;         // [n_mats, D, D] its noise matrix sqrt(C - c1 C c1^T)
    int64_t gle_stride;           // 0 (one matrix for every mode) or D * D (one per mode)
    int64_t n_atoms;
    double pos_conv;
    double dt;                    // time step (OP_BARO)
    double kbt_p;                 // P kB T (OP_PILE)
    uint64_t seed;
    int32_t P;
    int32_t global;
    int32_t gle_d;                // D (OP_GLE)
    spk_nhc_params_t q;           // (OP_NHC)
};

struct Workspace {
    double* sys_part;  // [n_sys, RP_NV]
    double* tot;       // [n_sys, RP_NV]
    double* head;      // [n_blocks, RP_NV]
};

static inline int64_t rp_blocks(int64_t n_atoms) { return spk_cdiv(n_atoms, RP_KT); }

static inline Workspace carve(void* ws, int64_t n_sys) {
    double* d = reinterpret_cast<double*>(ws);
    return Workspace{d, d + RP_NV * n_sys, d + 2 * RP_NV * n_sys};
}

static inline size_t mode_smem(int P) { return (size_t)P * RP_T * (2 * sizeof(double) + 2 * sizeof(float)); }

// normal d (0, 1, 2 = x, y, z) of the draw for element elem: the first three Box-Muller normals, as k_langevin
__device__ __forceinline__ double mode_noise(uint64_t seed, uint64_t app, int64_t elem, int d) {
    const uint4 r = philox_draw(seed, app, elem);
    if (d == 2) return box_muller(r.z, r.w).x;
    const double2 z = box_muller(r.x, r.y);
    return d == 0 ? z.x : z.y;
}

// PILE-G centroid factor of system s (thermostats_rpmd.py:160-195) with R = the x-noise of the system's own first atom;
// a system whose centroid kinetic energy is zero keeps its centroid (alpha = 1)
__device__ __forceinline__ double pile_alpha(const RpmdArgs& A, uint64_t app, int64_t s) {
    const double k0 = A.tot[RP_NV * s], S = A.tot[RP_NV * s + 1];
    if (!(k0 > 0.0)) return 1.0;
    const double c = A.c1[0];
    const double factor = k0 / A.kbt_p;                                         // :167-169
    const double cf = (1.0 - c) / factor;                                       // :171
    const double R = mode_noise(A.seed, app, A.sys_ptr[s], 0);
    const double a2 = c + S * cf + 2.0 * R * sqrt(c * cf);                      // :173-181
    const double sg = R + sqrt(c / cf);                                         // :183-186 torch.sign
    return sqrt(a2) * (double)((sg > 0.0) - (sg < 0.0));
}

// noise column c of the GLE row (mode k, dof i of atom a): normal d of the Philox draw of element (c P + k) N + a
__device__ __forceinline__ double gle_noise(const RpmdArgs& A, uint64_t app, int c, int k, int64_t a, int d) {
    return mode_noise(A.seed, app, ((int64_t)c * A.P + k) * A.n_atoms + a, d);
}

// one GLE application to the row (mode k, dof i): s[0] = p~, s <- c1_k s + sqrt(m) c2_k xi (Ceriotti, Bussi, Parrinello
// 2010, column-vector form; the reference multiplies the row vector s c1 = c1^T s, see DESIGN.md section 9); returns the
// new p~ = s[0].  D <= GLE_MAX_D is a run-time value: the loops are unrolled to GLE_MAX_D with guards, so s stays in
// registers, and threads of a warp share k, so the matrix reads are broadcasts.
__device__ __forceinline__ double gle_step(const RpmdArgs& A, uint64_t app, int k, int64_t i, int64_t a, double ma,
                                           double pn) {
    const int D = A.gle_d;
    const double* c1 = A.gle_c1 + k * A.gle_stride;
    const double* c2 = A.gle_c2 + k * A.gle_stride;
    double* row = A.gle_s + ((int64_t)k * 3 * A.n_atoms + i) * D;
    const int d = (int)(i - 3 * a);
    double s[GLE_MAX_D], acc[GLE_MAX_D];
#pragma unroll
    for (int c = 0; c < GLE_MAX_D; ++c) {
        s[c] = c == 0 ? pn : (c < D ? row[c] : 0.0);                   // thermostats.py:720
        acc[c] = 0.0;
    }
#pragma unroll
    for (int c = 0; c < GLE_MAX_D; ++c) {                              // c2 xi, one noise column at a time
        if (c < D) {
            const double xi = gle_noise(A, app, c, k, a, d);
#pragma unroll
            for (int r = 0; r < GLE_MAX_D; ++r)
                if (r < D) acc[r] += c2[r * D + c] * xi;
        }
    }
    const double sm = sqrt(ma);
#pragma unroll
    for (int r = 0; r < GLE_MAX_D; ++r) {
        if (r < D) {
            double v = 0.0;
#pragma unroll
            for (int c = 0; c < GLE_MAX_D; ++c)
                if (c < D) v += c1[r * D + c] * s[c];
            acc[r] = v + sm * acc[r];
            row[r] = acc[r];
        }
    }
    return acc[0];
}

// beads -> normal modes, the per-mode operator OP, normal modes -> beads, for RP_T degrees of freedom per CTA
template <int OP>
__global__ void __launch_bounds__(RP_THREADS) k_rpmd_modes(const __grid_constant__ RpmdArgs A) {
    constexpr bool HAS_X = OP == OP_MAIN || OP == OP_BARO;
    constexpr bool HAS_NOISE = OP == OP_PILE || OP == OP_GLE;
    extern __shared__ double smem[];
    const int P = A.P;
    const int PT = P * RP_T;
    double* mx = smem;                                   // [P][RP_T] normal modes of x
    double* mp = smem + PT;                              // [P][RP_T] normal modes of p
    float* bx = reinterpret_cast<float*>(smem + 2 * PT); // [P][RP_T] bead values
    float* bp = bx + PT;
    SPK_PDL_ENTER();
    unsigned long long app = 0;
    if (HAS_NOISE) app = *(volatile unsigned long long*)A.counter;
    const int64_t n_dof = 3 * A.n_atoms;
    const int64_t i0 = (int64_t)blockIdx.x * RP_T;
    for (int j = threadIdx.x; j < PT; j += RP_THREADS) {
        const int b = j / RP_T;
        const int64_t i = i0 + (j % RP_T);
        if (i < n_dof) {
            if (HAS_X) bx[j] = A.x[b * n_dof + i];
            bp[j] = A.p[b * n_dof + i];
        }
    }
    __syncthreads();
    for (int j = threadIdx.x; j < PT; j += RP_THREADS) {
        const int k = j / RP_T, t = j % RP_T;
        const int64_t i = i0 + t;
        if (i >= n_dof) continue;
        const double* Ck = A.C + (int64_t)k * P;
        double xn = 0.0, pn = 0.0;
        for (int b = 0; b < P; ++b) {                    // normal_model_transformation.py:78-80 beads2normal
            const double c = Ck[b];
            if (HAS_X) xn += c * (double)bx[b * RP_T + t];
            pn += c * (double)bp[b * RP_T + t];
        }
        const int64_t a = i / 3;
        const double ma = (double)A.m[a];
        if (OP == OP_BARO && k == 0) {                   // barostats_rpmd.py:136-143: the scaled p~_0 drives x~_0
            const double* ab = A.baro_ab + 2 * A.idx_m[a];
            pn = pn * ab[0];
            xn = xn / ab[0] + ab[1] * (pn / ma) * A.dt;
        } else if (HAS_X) {                              // integrators.py:221-230, barostats_rpmd.py:152-160
            const double* u = A.prop + 4 * k;
            const double np = u[0] * pn + u[1] * xn * ma;
            xn = u[2] * pn / ma + u[3] * xn;
            pn = np;
        } else if (OP == OP_PILE) {
            if (k == 0 && A.global) {                    // thermostats_rpmd.py:188-189
                pn *= pile_alpha(A, app, A.idx_m[a]);
            } else {                                     // :115-119, :191-195
                const double xi = mode_noise(A.seed, app, (int64_t)k * A.n_atoms + a, (int)(i - 3 * a));
                pn = A.c1[k] * pn + sqrt(ma * A.kbt_p) * A.c2[k] * xi;
            }
        } else if (OP == OP_GLE) {                       // thermostats.py:705-729, thermostats_rpmd.py:271-295
            pn = gle_step(A, app, k, i, a, ma, pn);
        } else {                                         // thermostats_rpmd.py:465-501
            double ke = pn * pn / ma, dof = 1.0;
            if (k == 0 && A.global) {
                const int64_t s = A.idx_m[a];
                ke = A.tot[RP_NV * s];
                dof = 3.0 * (double)(A.sys_ptr[s + 1] - A.sys_ptr[s]);
            }
            const int L = A.q.chain_length;
            const int64_t row = (int64_t)k * n_dof + i;
            pn *= nhc_propagate(ke, dof, A.q, A.q.kb_temperature, A.chain_v + row * L, A.chain_f + row * L,
                                A.chain_m + row * L);
        }
        if (HAS_X) mx[j] = xn;
        mp[j] = pn;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < PT; j += RP_THREADS) {
        const int b = j / RP_T, t = j % RP_T;
        const int64_t i = i0 + t;
        if (i >= n_dof) continue;
        double xb = 0.0, pb = 0.0;
        for (int k = 0; k < P; ++k) {                    // normal_model_transformation.py:93-101 normal2beads
            const double c = A.C[(int64_t)k * P + b];
            if (HAS_X) xb += c * mx[k * RP_T + t];
            pb += c * mp[k * RP_T + t];
        }
        A.p[b * n_dof + i] = (float)pb;
        if (HAS_X) {
            const float xf = (float)xb;
            A.x[b * n_dof + i] = xf;
            if (A.model_x) A.model_x[b * n_dof + i] = xf * (float)A.pos_conv;
        }
    }
    if (HAS_NOISE) advance_counter(A.counter, app);
}

// free-particle-limit start of the GLE state (thermostats.py:687-701): the row vector s = xi c2_k, without a mass factor,
// one thread per (mode k, dof i); noise as gle_step at the current application
__global__ void __launch_bounds__(RP_THREADS) k_gle_init(const __grid_constant__ RpmdArgs A) {
    SPK_PDL_ENTER();
    const unsigned long long app = *(volatile unsigned long long*)A.counter;
    const int64_t n_dof = 3 * A.n_atoms;
    const int64_t rowi = (int64_t)blockIdx.x * RP_THREADS + threadIdx.x;
    if (rowi < (int64_t)A.P * n_dof) {
        const int k = (int)(rowi / n_dof);
        const int64_t i = rowi - (int64_t)k * n_dof, a = i / 3;
        const int D = A.gle_d;
        const double* c2 = A.gle_c2 + k * A.gle_stride;
        double acc[GLE_MAX_D];
#pragma unroll
        for (int c = 0; c < GLE_MAX_D; ++c) acc[c] = 0.0;
#pragma unroll
        for (int j = 0; j < GLE_MAX_D; ++j) {
            if (j < D) {
                const double xi = gle_noise(A, app, j, k, a, (int)(i - 3 * a));
#pragma unroll
                for (int c = 0; c < GLE_MAX_D; ++c)
                    if (c < D) acc[c] += xi * c2[j * D + c];
            }
        }
        double* row = A.gle_s + rowi * D;
#pragma unroll
        for (int c = 0; c < GLE_MAX_D; ++c)
            if (c < D) row[c] = acc[c];
    }
    advance_counter(A.counter, app);
}

// out = C in (inverse = 0) or C^T in (inverse = 1) over the bead axis, RP_T degrees of freedom per CTA
__global__ void __launch_bounds__(RP_THREADS) k_rpmd_transform(const float* in, float* out, int64_t n_dof, int P,
                                                             const double* __restrict__ C, int inverse) {
    extern __shared__ double smem[];
    float* bv = reinterpret_cast<float*>(smem);          // [P][RP_T]
    SPK_PDL_ENTER();
    const int PT = P * RP_T;
    const int64_t i0 = (int64_t)blockIdx.x * RP_T;
    for (int j = threadIdx.x; j < PT; j += RP_THREADS) {
        const int64_t i = i0 + (j % RP_T);
        if (i < n_dof) bv[j] = in[(j / RP_T) * n_dof + i];
    }
    __syncthreads();
    for (int j = threadIdx.x; j < PT; j += RP_THREADS) {
        const int r = j / RP_T, t = j % RP_T;
        const int64_t i = i0 + t;
        if (i >= n_dof) continue;
        double acc = 0.0;
        for (int q = 0; q < P; ++q) acc += (inverse ? C[q * P + r] : C[r * P + q]) * (double)bv[q * RP_T + t];
        out[r * n_dof + i] = (float)acc;
    }
}

// per-(system, CTA) partials of sum_a |p~_0,a|^2 / m_a and (with_noise) sum_a |xi_0,a|^2 over the atoms of the base batch
__global__ void __launch_bounds__(RP_KT) k_rpmd_centroid_partials(const __grid_constant__ RpmdArgs A, int with_noise,
                                                                  double* __restrict__ sys_part,
                                                                  double* __restrict__ head) {
    SPK_PDL_ENTER();
    const unsigned long long app = with_noise ? *(volatile unsigned long long*)A.counter : 0ull;
    const int64_t a = (int64_t)blockIdx.x * RP_KT + threadIdx.x;
    const int64_t n_dof = 3 * A.n_atoms;
    double v[RP_NV] = {0.0, 0.0};
    int64_t s = 0, first = 0, end = 0;
    if (a < A.n_atoms) {
        const double ma = (double)A.m[a];
        for (int d = 0; d < 3; ++d) {
            double pc = 0.0;
            for (int b = 0; b < A.P; ++b) pc += A.C[b] * (double)A.p[b * n_dof + 3 * a + d];   // row 0 of C
            v[0] += pc * pc / ma;                                                        // thermostats_rpmd.py:162-165
        }
        if (with_noise) {
            const uint4 r = philox_draw(A.seed, app, a);
            const double2 z01 = box_muller(r.x, r.y), z23 = box_muller(r.z, r.w);
            v[1] = z01.x * z01.x + z01.y * z01.y + z23.x * z23.x;                        // :174-176
        }
        s = A.idx_m[a];
        first = A.sys_ptr[s];
        end = A.sys_ptr[s + 1];
    }
    seg_partials<RP_KT, RP_NV>(v, A.n_atoms, s, first, end, sys_part, head);
}

// ---- PILE barostat (barostats_rpmd.py) -----------------------------------------------------------------------------------
struct BaroArgs {
    const float* p;               // bead momenta [P, n_atoms, 3]
    const float* f;               // bead forces [P, n_atoms, 3], model units (times f_conv)
    const float* m;               // [n_atoms]
    const int64_t* idx_m;         // base batch
    const int32_t* sys_ptr;
    const double* C;              // [P, P]
    const double* cell;           // [P n_sys, 3, 3] MD cells of the bead systems
    const double* virial;         // [P n_sys, 3, 3] model-unit virials of the bead systems
    const double* W;              // [n_sys] cell masses
    double* pc;                   // [n_sys] cell momenta
    int64_t n_atoms;
    int64_t n_sys;
    double f_conv;
    double virial_scale;          // stress = virial_scale * virial / det(cell)
    double target_pressure;
    double kbt;
    double dt;
    int32_t P;
};

struct BaroWorkspace {
    double* sys_part;  // [n_sys, RB_NV]
    double* ab;        // [n_sys, 2]
    double* head;      // [n_blocks, RB_NV]
};

static inline BaroWorkspace carve_baro(void* ws, int64_t n_sys) {
    double* d = reinterpret_cast<double*>(ws);
    return BaroWorkspace{d, d + RB_NV * n_sys, d + (RB_NV + 2) * n_sys};
}

// _update_barostat (barostats_rpmd.py:101-110): p_c = c1 p_c + c2[s] xi, one thread per system; xi is normal 0 of the
// Philox draw (seed; counter = system, application), and the application index advances by advance_counter
__global__ void k_rpmd_baro_pile(double* __restrict__ pc, int64_t n_sys, double c1, const double* __restrict__ c2,
                                 uint64_t seed, unsigned long long* counter) {
    SPK_PDL_ENTER();
    const unsigned long long app = *(volatile unsigned long long*)counter;
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s < n_sys) {
        const uint4 r = philox_draw(seed, app, s);
        pc[s] = c1 * pc[s] + c2[s] * box_muller(r.x, r.y).x;
    }
    advance_counter(counter, app);
}

// propagate_half_step (barostats_rpmd.py:173-199), per-(system, CTA) partials over the base atoms: mode 0 of the forces
// (MD units) and momenta, one row of C across the P beads, and the bead mean of the momenta
__global__ void __launch_bounds__(RP_KT) k_rpmd_baro_partials(const __grid_constant__ BaroArgs B,
                                                              double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * RP_KT + threadIdx.x;
    const int64_t n_dof = 3 * B.n_atoms;
    double v[RB_NV] = {0.0, 0.0, 0.0};
    int64_t s = 0, first = 0, end = 0;
    if (a < B.n_atoms) {
        const double ma = (double)B.m[a];
        double pm2 = 0.0;
        for (int d = 0; d < 3; ++d) {
            double p0 = 0.0, f0 = 0.0, ps = 0.0;
            for (int b = 0; b < B.P; ++b) {
                const int64_t i = b * n_dof + 3 * a + d;
                const double pb = (double)B.p[i];
                p0 += B.C[b] * pb;
                f0 += B.C[b] * ((double)B.f[i] * B.f_conv);
                ps += pb;
            }
            const double fm = f0 / ma;                   // :180
            v[0] += fm * p0;                             // :182-184
            v[1] += fm * f0 / 3.0;                       // :185-187
            const double pm = ps / (double)B.P;          // system.py:497-508, 524-537
            pm2 += pm * pm;
        }
        v[2] = pm2 / ma;
        s = B.idx_m[a];
        first = B.sys_ptr[s];
        end = B.sys_ptr[s + 1];
    }
    seg_partials<RP_KT, RB_NV>(v, B.n_atoms, s, first, end, sys_part, head);
}

// one CTA per system: the ordered total of the partials, then (thread 0) the centroid pressure from the bead means of the
// volume and stress (system.py:616-650) and p_c += h c1 + h^2 c2 + h^3 c3 with h = dt / 2 (barostats_rpmd.py:164-205)
__global__ void __launch_bounds__(SEG_FIN_T) k_rpmd_baro_finish(const __grid_constant__ BaroArgs B,
                                                                const double* __restrict__ sys_part,
                                                                const double* __restrict__ head) {
    __shared__ double red[RB_NV][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x;
    seg_finish_block<RP_KT, RB_NV>(B.sys_ptr, nullptr, sys_part, head, s, red);
    if (threadIdx.x != 0) return;
    double vsum = 0.0, st[3] = {0.0, 0.0, 0.0};
    for (int r = 0; r < B.P; ++r) {
        const int64_t bs = (int64_t)r * B.n_sys + s;
        const double V = det3(B.cell + 9 * bs);
        vsum += V;
        for (int k = 0; k < 3; ++k) st[k] += B.virial_scale * B.virial[9 * bs + 4 * k] / V;
    }
    const double inv_p = 1.0 / (double)B.P;
    const double vbar = vsum * inv_p;
    const double p_vir = ((-st[0] * inv_p) + (-st[1] * inv_p) + (-st[2] * inv_p)) / 3.0;
    const double p_cent = p_vir + 2.0 * (0.5 * red[2][0]) / vbar / 3.0;
    const double c1 = 3.0 * (double)B.P * (vbar * (p_cent - B.target_pressure) + B.kbt);
    const double h = 0.5 * B.dt;
    B.pc[s] = B.pc[s] + (h * c1 + (h * h) * red[0][0] + (h * h * h) * red[1][0]);
}

// propagate_main_step (barostats_rpmd.py:119-133), one thread per system: (a, b) = (exp(-dt p_c / W), StableSinhDiv(dt
// p_c / W)) for the mode kernel, and every bead copy of the cell divided by a (model cell = MD cell * position_conversion)
__global__ void k_rpmd_baro_cell(const double* __restrict__ pc, const double* __restrict__ W, int64_t n_sys, int P,
                                 double dt, double* __restrict__ cell, float* __restrict__ model_cell, double pos_conv,
                                 double* __restrict__ ab) {
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_sys) return;
    const double x = dt * (pc[s] / W[s]);
    const double a = exp(-x);
    ab[2 * s] = a;
    ab[2 * s + 1] = stable_sinh_div(x);
    for (int r = 0; r < P; ++r) {
        const int64_t bs = (int64_t)r * n_sys + s;
        for (int k = 0; k < 9; ++k) {
            const double c = cell[9 * bs + k] / a;
            cell[9 * bs + k] = c;
            if (model_cell) model_cell[9 * bs + k] = (float)(c * pos_conv);
        }
    }
}

static bool beads_ok(int P, const double* C) { return P >= 1 && P <= RP_MAX_BEADS && C; }

static int check_modes(const float* momenta, const float* masses, int64_t n_atoms, int P, const double* C) {
    if (!beads_ok(P, C) || n_atoms < 0 || (int64_t)P * 3 * n_atoms >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!momenta || !masses)) return SPK_ERR_ARG;
    return SPK_OK;
}

static int check_systems(const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, void* workspace,
                         size_t workspace_bytes) {
    if (n_sys <= 0 || !sys_ptr || (n_atoms > 0 && !idx_m)) return SPK_ERR_ARG;
    if (!workspace || workspace_bytes < spk_rpmd_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    return SPK_OK;
}

template <int OP>
static void launch_modes(const RpmdArgs& A, cudaStream_t st) {
    spk_launch(k_rpmd_modes<OP>, (unsigned)spk_cdiv(3 * A.n_atoms, RP_T), RP_THREADS, mode_smem(A.P), st, A);
}

// the per-system centroid sums of the global variants: partials + ordered per-system finish (2 launches)
static void centroid_sums(RpmdArgs& A, int with_noise, int64_t n_sys, void* workspace, cudaStream_t st) {
    Workspace w = carve(workspace, n_sys);
    spk_launch(k_rpmd_centroid_partials, (unsigned)rp_blocks(A.n_atoms), RP_KT, 0, st, A, with_noise, w.sys_part,
               w.head);
    spk_launch(k_seg_finish<RP_KT, RP_NV>, (unsigned)n_sys, SEG_FIN_T, 0, st, A.sys_ptr, (const int32_t*)nullptr,
               (const double*)w.sys_part, (const double*)w.head, w.tot);
    A.tot = w.tot;
}

}  // namespace

extern "C" size_t spk_rpmd_barostat_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? rp_blocks(n_atoms) : 0;
    return sizeof(double) * (size_t)((RB_NV + 2) * (n_sys > 0 ? n_sys : 0) + RB_NV * nb + 1);
}

extern "C" size_t spk_rpmd_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? rp_blocks(n_atoms) : 0;
    return sizeof(double) * (size_t)(RP_NV * (2 * (n_sys > 0 ? n_sys : 0) + nb) + 1);
}

extern "C" int spk_rpmd_normal_modes(const float* in, float* out, int64_t n_atoms, int32_t n_beads,
                                     const double* c_transform, int32_t inverse, spk_stream_t stream) {
    if (!beads_ok(n_beads, c_transform) || n_atoms < 0 || (int64_t)n_beads * 3 * n_atoms >= (1ll << 31) - 1)
        return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!in || !out) return SPK_ERR_ARG;
    spk_launch(k_rpmd_transform, (unsigned)spk_cdiv(3 * n_atoms, RP_T), RP_THREADS,
               (size_t)n_beads * RP_T * sizeof(float), spk_st(stream), in, out, 3 * n_atoms, (int)n_beads, c_transform,
               inverse ? 1 : 0);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_main_step(float* positions, float* momenta, float* model_positions, const float* masses,
                                  int64_t n_atoms, int32_t n_beads, const double* c_transform, const double* propagator,
                                  double position_conversion, spk_stream_t stream) {
    if (check_modes(momenta, masses, n_atoms, n_beads, c_transform) != SPK_OK || !propagator) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!positions) return SPK_ERR_ARG;
    RpmdArgs A = {};
    A.x = positions;
    A.p = momenta;
    A.model_x = model_positions;
    A.m = masses;
    A.C = c_transform;
    A.prop = propagator;
    A.n_atoms = n_atoms;
    A.pos_conv = position_conversion;
    A.P = n_beads;
    launch_modes<OP_MAIN>(A, spk_st(stream));
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_pile(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                             int64_t n_atoms, int64_t n_sys, int32_t n_beads, const double* c_transform, const double* c1,
                             const double* c2, double kb_temperature, int32_t global, uint64_t seed, uint64_t* counter,
                             void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (check_modes(momenta, masses, n_atoms, n_beads, c_transform) != SPK_OK) return SPK_ERR_ARG;
    if (!c1 || !c2 || !counter || !(kb_temperature > 0.0)) return SPK_ERR_ARG;
    if (global && check_systems(idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes) != SPK_OK)
        return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    cudaStream_t st = spk_st(stream);
    RpmdArgs A = {};
    A.p = momenta;
    A.m = masses;
    A.idx_m = idx_m;
    A.sys_ptr = sys_ptr;
    A.C = c_transform;
    A.c1 = c1;
    A.c2 = c2;
    A.counter = reinterpret_cast<unsigned long long*>(counter);
    A.n_atoms = n_atoms;
    A.kbt_p = kb_temperature;
    A.seed = seed;
    A.P = n_beads;
    A.global = global ? 1 : 0;
    if (A.global) centroid_sums(A, 1, n_sys, workspace, st);
    launch_modes<OP_PILE>(A, st);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_nhc(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                            int64_t n_atoms, int64_t n_sys, int32_t n_beads, const double* c_transform,
                            const spk_nhc_params_t* params, int32_t global, double* chain_v, double* chain_f,
                            const double* chain_m, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (check_modes(momenta, masses, n_atoms, n_beads, c_transform) != SPK_OK) return SPK_ERR_ARG;
    if (!params || params->chain_length < 1 || params->multi_step < 1 ||
        !(params->order == 3 || params->order == 5 || params->order == 7) || !(params->kb_temperature > 0.0))
        return SPK_ERR_ARG;
    if (!chain_v || !chain_f || !chain_m) return SPK_ERR_ARG;
    if (global && check_systems(idx_m, sys_ptr, n_atoms, n_sys, workspace, workspace_bytes) != SPK_OK)
        return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    cudaStream_t st = spk_st(stream);
    RpmdArgs A = {};
    A.p = momenta;
    A.m = masses;
    A.idx_m = idx_m;
    A.sys_ptr = sys_ptr;
    A.C = c_transform;
    A.chain_v = chain_v;
    A.chain_f = chain_f;
    A.chain_m = chain_m;
    A.n_atoms = n_atoms;
    A.P = n_beads;
    A.global = global ? 1 : 0;
    A.q = *params;
    if (A.global) centroid_sums(A, 0, n_sys, workspace, st);
    launch_modes<OP_NHC>(A, st);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_gle(float* momenta, const float* masses, int64_t n_atoms, int32_t n_beads,
                            const double* c_transform, const double* c1, const double* c2, int32_t gle_dim,
                            int32_t per_mode, double* state, uint64_t seed, uint64_t* counter, int32_t initial,
                            spk_stream_t stream) {
    if (!beads_ok(n_beads, c_transform) || n_atoms < 0 || (int64_t)n_beads * 3 * n_atoms >= (1ll << 31) - 1)
        return SPK_ERR_ARG;
    if (n_atoms > 0 && !initial && (!momenta || !masses)) return SPK_ERR_ARG;   // the initial draw reads neither
    if (gle_dim < 1 || gle_dim > GLE_MAX_D || !c1 || !c2 || !state || !counter) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    RpmdArgs A = {};
    A.p = momenta;
    A.m = masses;
    A.C = c_transform;
    A.gle_s = state;
    A.gle_c1 = c1;
    A.gle_c2 = c2;
    A.gle_stride = per_mode ? (int64_t)gle_dim * gle_dim : 0;
    A.gle_d = gle_dim;
    A.counter = reinterpret_cast<unsigned long long*>(counter);
    A.n_atoms = n_atoms;
    A.seed = seed;
    A.P = n_beads;
    cudaStream_t st = spk_st(stream);
    if (initial)
        spk_launch(k_gle_init, (unsigned)spk_cdiv((int64_t)n_beads * 3 * n_atoms, RP_THREADS), RP_THREADS, 0, st, A);
    else
        launch_modes<OP_GLE>(A, st);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_barostat_thermostat(double* cell_momenta, int64_t n_sys, double c1, const double* c2, uint64_t seed,
                                            uint64_t* counter, spk_stream_t stream) {
    if (n_sys <= 0 || !cell_momenta || !c2 || !counter) return SPK_ERR_ARG;
    spk_launch(k_rpmd_baro_pile, (unsigned)spk_cdiv(n_sys, 128), 128, 0, spk_st(stream), cell_momenta, n_sys, c1, c2,
               seed, reinterpret_cast<unsigned long long*>(counter));
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_barostat_half_step(const float* momenta, const float* forces, double force_conversion,
                                           const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                                           int64_t n_atoms, int64_t n_sys, int32_t n_beads, const double* c_transform,
                                           const double* cells, const double* virial, double virial_scale,
                                           double target_pressure, double kb_temperature, double time_step,
                                           const double* cell_mass, double* cell_momenta, void* workspace,
                                           size_t workspace_bytes, spk_stream_t stream) {
    if (check_modes(momenta, masses, n_atoms, n_beads, c_transform) != SPK_OK) return SPK_ERR_ARG;
    if (n_sys <= 0 || !sys_ptr || (n_atoms > 0 && (!idx_m || !forces))) return SPK_ERR_ARG;
    if (!cells || !virial || !cell_mass || !cell_momenta || !workspace ||
        workspace_bytes < spk_rpmd_barostat_workspace_bytes(n_atoms, n_sys))
        return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    const BaroWorkspace w = carve_baro(workspace, n_sys);
    BaroArgs B = {};
    B.p = momenta;
    B.f = forces;
    B.m = masses;
    B.idx_m = idx_m;
    B.sys_ptr = sys_ptr;
    B.C = c_transform;
    B.cell = cells;
    B.virial = virial;
    B.W = cell_mass;
    B.pc = cell_momenta;
    B.n_atoms = n_atoms;
    B.n_sys = n_sys;
    B.f_conv = force_conversion;
    B.virial_scale = virial_scale;
    B.target_pressure = target_pressure;
    B.kbt = kb_temperature;
    B.dt = time_step;
    B.P = n_beads;
    if (n_atoms > 0)
        spk_launch(k_rpmd_baro_partials, (unsigned)rp_blocks(n_atoms), RP_KT, 0, st, B, w.sys_part, w.head);
    spk_launch(k_rpmd_baro_finish, (unsigned)n_sys, SEG_FIN_T, 0, st, B, (const double*)w.sys_part,
               (const double*)w.head);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rpmd_barostat_main_step(float* positions, float* momenta, float* model_positions, const float* masses,
                                           const int64_t* idx_m, int64_t n_atoms, int64_t n_sys, int32_t n_beads,
                                           const double* c_transform, const double* propagator, double time_step,
                                           const double* cell_momenta, const double* cell_mass, double* cells,
                                           float* model_cells, double position_conversion, void* workspace,
                                           size_t workspace_bytes, spk_stream_t stream) {
    if (check_modes(momenta, masses, n_atoms, n_beads, c_transform) != SPK_OK || !propagator) return SPK_ERR_ARG;
    if (n_sys <= 0 || !cells || !cell_momenta || !cell_mass || (n_atoms > 0 && (!positions || !idx_m))) return SPK_ERR_ARG;
    if (!workspace || workspace_bytes < spk_rpmd_barostat_workspace_bytes(n_atoms, n_sys)) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    const BaroWorkspace w = carve_baro(workspace, n_sys);
    spk_launch(k_rpmd_baro_cell, (unsigned)spk_cdiv(n_sys, 128), 128, 0, st, cell_momenta, cell_mass, n_sys,
               (int)n_beads, time_step, cells, model_cells, position_conversion, w.ab);
    if (n_atoms > 0) {
        RpmdArgs A = {};
        A.x = positions;
        A.p = momenta;
        A.model_x = model_positions;
        A.m = masses;
        A.idx_m = idx_m;
        A.C = c_transform;
        A.prop = propagator;
        A.baro_ab = w.ab;
        A.n_atoms = n_atoms;
        A.pos_conv = position_conversion;
        A.dt = time_step;
        A.P = n_beads;
        launch_modes<OP_BARO>(A, st);
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

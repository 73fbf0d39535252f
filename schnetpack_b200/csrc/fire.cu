// Batchwise FIRE relaxation on the device (ASE's FIRE without downhill_check), one independent optimizer per system of a
// collated batch, optionally on the generalized coordinates of ASE's UnitCellFilter; all optimizer state is fp64.
//
// A FIRE step needs three per-system dot products (v.g, v.v, g.g) and the convergence test a per-system max, so the
// whole optimizer is five bandwidth-bound launches around the model:
//   force side (spk_fire_forces, after every evaluation):
//     k_fire_atoms   one thread per atom: g_i = f_i F (0 on fixed atoms) and the (system, CTA) partials of the three
//                    dot products (seg_partials of segscan.cuh);
//     k_fire_system  one CTA per system: the partials in CTA order, the 3 cell rows of g (filter), the largest row
//                    |g_row|^2, the convergence test;
//     k_count_unconverged  the count of unconverged systems (relax_common.cuh);
//   step (spk_fire_step):
//     k_fire_coef    one thread per system: dt, a, Nsteps, the cap of |dr| and the cell's 9 components (it owns them);
//     k_fire_move    one thread per atom: v, s, x = s F^T and the fp32 model positions.
// |v'|^2 after the mixing follows from v.v, v.g and g.g (v' = c1 v + c2 g with c1, c2 >= 0), so no second reduction pass
// is needed.  Every sum has a fixed order given the layout and there are no atomics: replays are bitwise reproducible.
#include "relax_common.cuh"
#include "segscan.cuh"

namespace {

constexpr int FIRE_T = 256;      // atoms per CTA of the partial pass
constexpr int NSUM = 3;          // v.g, v.v, g.g
constexpr int MOVE_T = 256;
constexpr int COEF_T = 128;

// coefficients the per-system thread leaves for k_fire_move, [n_sys][COEF_N]
enum { C_MODE = 0, C_ONE_MINUS_A, C_A, C_GNORM, C_VNORM, C_DT, C_NORMDR, COEF_N };
enum { MODE_FROZEN = 0, MODE_START = 1, MODE_MIX = 2, MODE_RESET = 3 };

// F = h / cell_factor of system m, row-major [3][3]
__device__ __forceinline__ void load_F(const spk_fire_t& st, int64_t m, double (&F)[9]) {
    const double cf = st.cell_factor[m];
#pragma unroll
    for (int k = 0; k < 9; ++k) F[k] = st.h[9 * m + k] / cf;
}

// f_i F (row vector times F), in optimizer units, 0 on fixed atoms
__device__ __forceinline__ void atom_force(const spk_fire_t& st, const float* __restrict__ forces, int64_t a, int64_t m,
                                           double (&g)[3]) {
    const bool fixed = st.fixed && st.fixed[a];
    double f[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) f[c] = optimizer_force(fixed, forces, st.force_conversion, a, c);
    if (!st.filter) {
#pragma unroll
        for (int c = 0; c < 3; ++c) g[c] = f[c];
        return;
    }
    double F[9];
    load_F(st, m, F);
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = dot3_rn(f[0], f[1], f[2], F[k], F[3 + k], F[6 + k]);
}

__device__ __forceinline__ double* ws_sys_part(const spk_fire_t& st) { return st.workspace; }
__device__ __forceinline__ double* ws_head(const spk_fire_t& st) { return st.workspace + NSUM * st.n_sys; }

__global__ void __launch_bounds__(FIRE_T) k_fire_atoms(spk_fire_t st, const float* __restrict__ forces) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * FIRE_T + threadIdx.x;
    double v[NSUM] = {0.0, 0.0, 0.0};
    int64_t m = 0, first = 0, end = 0;
    if (a < st.n_atoms) {
        m = st.idx_m[a];
        first = st.sys_ptr[m];
        end = st.sys_ptr[m + 1];
        double g[3];
        atom_force(st, forces, a, m, g);
        const double v0 = st.v[3 * a], v1 = st.v[3 * a + 1], v2 = st.v[3 * a + 2];
#pragma unroll
        for (int c = 0; c < 3; ++c) st.g[3 * a + c] = g[c];
        v[0] = dot3_rn(v0, v1, v2, g[0], g[1], g[2]);
        v[1] = dot3_rn(v0, v1, v2, v0, v1, v2);
        v[2] = dot3_rn(g[0], g[1], g[2], g[0], g[1], g[2]);
    }
    seg_partials<FIRE_T, NSUM>(v, st.n_atoms, m, first, end, ws_sys_part(st), ws_head(st));
}

// 3x3 inverse by the adjugate (row-major)
__device__ __forceinline__ void inv3(const double (&A)[9], double (&B)[9]) {
    const double c00 = A[4] * A[8] - A[5] * A[7], c01 = A[5] * A[6] - A[3] * A[8], c02 = A[3] * A[7] - A[4] * A[6];
    const double det = A[0] * c00 + A[1] * c01 + A[2] * c02;
    const double id = 1.0 / det;
    B[0] = c00 * id;
    B[1] = (A[2] * A[7] - A[1] * A[8]) * id;
    B[2] = (A[1] * A[5] - A[2] * A[4]) * id;
    B[3] = c01 * id;
    B[4] = (A[0] * A[8] - A[2] * A[6]) * id;
    B[5] = (A[2] * A[3] - A[0] * A[5]) * id;
    B[6] = c02 * id;
    B[7] = (A[1] * A[6] - A[0] * A[7]) * id;
    B[8] = (A[0] * A[4] - A[1] * A[3]) * id;
}

// cell = cell0 F^T (rows = lattice vectors)
__device__ __forceinline__ void current_cell(const spk_fire_t& st, int64_t m, const double (&F)[9], double (&cell)[9]) {
    const double* c0 = st.cell0 + 9 * m;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            cell[3 * i + j] = dot3_rn(c0[3 * i], c0[3 * i + 1], c0[3 * i + 2], F[3 * j], F[3 * j + 1], F[3 * j + 2]);
}

// The generalized cell forces of UnitCellFilter.get_forces: Vir = -(energy_conversion sym(W) + p V I), Vir F^-T, the
// projections in ASE's order (hydrostatic_strain, mask, constant_volume), / cell_factor.
__device__ void cell_forces(const spk_fire_t& st, int64_t m, const double* __restrict__ virial, double (&hg)[9]) {
    double F[9], Fi[9], cell[9], vir[9], t[9];
    load_F(st, m, F);
    current_cell(st, m, F, cell);
    const double vol = fabs(cell[0] * (cell[4] * cell[8] - cell[5] * cell[7]) -
                            cell[1] * (cell[3] * cell[8] - cell[5] * cell[6]) +
                            cell[2] * (cell[3] * cell[7] - cell[4] * cell[6]));
    const double* W = virial + 9 * m;
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const double s = 0.5 * (W[3 * i + j] + W[3 * j + i]) * st.energy_conversion;
            vir[3 * i + j] = -(i == j ? s + st.scalar_pressure * vol : s);
        }
    inv3(F, Fi);
    // (Vir F^-T)_ij = sum_k Vir_ik Fi_jk
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            t[3 * i + j] = dot3_rn(vir[3 * i], vir[3 * i + 1], vir[3 * i + 2], Fi[3 * j], Fi[3 * j + 1], Fi[3 * j + 2]);
    if (st.hydrostatic_strain) {
        const double tr3 = (t[0] + t[4] + t[8]) / 3.0;
#pragma unroll
        for (int k = 0; k < 9; ++k) t[k] = (k % 4 == 0) ? tr3 : 0.0;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) t[k] *= st.mask[k];
    if (st.constant_volume) {
        const double tr3 = (t[0] + t[4] + t[8]) / 3.0;
        t[0] -= tr3;
        t[4] -= tr3;
        t[8] -= tr3;
    }
    const double cf = st.cell_factor[m];
#pragma unroll
    for (int k = 0; k < 9; ++k) hg[k] = t[k] / cf;
}

// One CTA per system: the dot products, the cell rows, fmax and the convergence test
__global__ void __launch_bounds__(SEG_FIN_T) k_fire_system(spk_fire_t st, const double* __restrict__ virial) {
    __shared__ double red[NSUM][SEG_FIN_T];
    __shared__ double mx_red[SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t m = blockIdx.x;
    const int t = threadIdx.x;
    seg_finish_block<FIRE_T, NSUM>(st.sys_ptr, nullptr, ws_sys_part(st), ws_head(st), m, red);
    // largest |g_row|^2 over the atom rows: strided over the CTA, then a fixed tree (max is exact in any order)
    const int64_t a0 = st.sys_ptr[m], a1 = st.sys_ptr[m + 1];
    double mx = 0.0;
    for (int64_t a = a0 + t; a < a1; a += SEG_FIN_T) {
        const double* g = st.g + 3 * a;
        mx = fmax(mx, dot3_rn(g[0], g[1], g[2], g[0], g[1], g[2]));
    }
    mx_red[t] = mx;
    __syncthreads();
#pragma unroll
    for (int d = SEG_FIN_T / 2; d > 0; d >>= 1) {
        if (t < d) mx_red[t] = fmax(mx_red[t], mx_red[t + d]);
        __syncthreads();
    }
    if (t != 0) return;
    double vg = red[0][0], vv = red[1][0], gg = red[2][0];
    mx = mx_red[0];
    if (st.filter) {
        double hg[9];
        cell_forces(st, m, virial, hg);
        const double* hv = st.hv + 9 * m;
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            const double* gr = hg + 3 * r;
            const double* vr = hv + 3 * r;
            vg += dot3_rn(vr[0], vr[1], vr[2], gr[0], gr[1], gr[2]);
            vv += dot3_rn(vr[0], vr[1], vr[2], vr[0], vr[1], vr[2]);
            const double g2 = dot3_rn(gr[0], gr[1], gr[2], gr[0], gr[1], gr[2]);
            gg += g2;
            mx = fmax(mx, g2);
        }
#pragma unroll
        for (int k = 0; k < 9; ++k) st.hg[9 * m + k] = hg[k];
    }
    st.sums[NSUM * m] = vg;
    st.sums[NSUM * m + 1] = vv;
    st.sums[NSUM * m + 2] = gg;
    record_convergence(st, m, mx);
}

// ASE's velocity update of one component: the mixing (or the reset) with the old a, then v += dt g with the new dt
__device__ __forceinline__ double new_velocity(const double* __restrict__ c, int mode, double v, double g) {
    if (mode == MODE_MIX) {
        const double mix = __dmul_rn(__ddiv_rn(__dmul_rn(c[C_A], g), c[C_GNORM]), c[C_VNORM]);
        v = __dadd_rn(__dmul_rn(c[C_ONE_MINUS_A], v), mix);
    } else if (mode == MODE_RESET) {
        v = 0.0;
    }
    return __dadd_rn(v, __dmul_rn(c[C_DT], g));
}

// dr = dt v, scaled to maxstep when |dr| over all the system's coordinates exceeds it
__device__ __forceinline__ double displacement(const spk_fire_t& st, const double* __restrict__ c, double v) {
    const double dr = __dmul_rn(c[C_DT], v);
    return c[C_NORMDR] > st.maxstep ? __ddiv_rn(__dmul_rn(st.maxstep, dr), c[C_NORMDR]) : dr;
}

// One thread per system: the FIRE scalars, |dr| from the three dot products, and the step of the 9 cell coordinates
__global__ void __launch_bounds__(COEF_T) k_fire_coef(spk_fire_t st) {
    SPK_PDL_ENTER();
    const int64_t m = (int64_t)blockIdx.x * COEF_T + threadIdx.x;
    if (blockIdx.x == 0 && threadIdx.x == 0) st.counter[1] = st.counter[0] + 1;
    if (m >= st.n_sys) return;
    double* c = st.coef + COEF_N * m;
    if (st.converged[m]) {
        c[C_MODE] = MODE_FROZEN;
        return;
    }
    const double vg = st.sums[NSUM * m], vv = st.sums[NSUM * m + 1], gg = st.sums[NSUM * m + 2];
    double dt = st.dt[m], a = st.a[m];
    int64_t ns = st.nsteps[m];
    int mode;
    double c1, c2;                       // v' = c1 v + c2 g
    const double vn = sqrt(vv), gn = sqrt(gg);
    if (!st.started[m]) {
        st.started[m] = 1;
        mode = MODE_START;
        c1 = 0.0;
        c2 = 0.0;
    } else if (vg > 0.0) {
        mode = MODE_MIX;
        c[C_ONE_MINUS_A] = 1.0 - a;
        c[C_A] = a;
        c1 = 1.0 - a;
        c2 = a * vn / gn;
        if (ns > st.nmin) {
            dt = fmin(dt * st.finc, st.dtmax);
            a *= st.fa;
        }
        ns += 1;
    } else {
        mode = MODE_RESET;
        c1 = 0.0;
        c2 = 0.0;
        a = st.astart;
        dt *= st.fdec;
        ns = 0;
    }
    c2 += dt;
    const double v2 = c1 * c1 * vv + 2.0 * c1 * c2 * vg + c2 * c2 * gg;
    c[C_MODE] = mode;
    c[C_GNORM] = gn;
    c[C_VNORM] = vn;
    c[C_DT] = dt;
    c[C_NORMDR] = dt * sqrt(v2);
    st.dt[m] = dt;
    st.a[m] = a;
    st.nsteps[m] = ns;
    if (!st.filter) return;
    double F[9], cell[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
        const double v = new_velocity(c, mode, st.hv[9 * m + k], st.hg[9 * m + k]);
        st.hv[9 * m + k] = v;
        st.h[9 * m + k] += displacement(st, c, v);
    }
    load_F(st, m, F);
    current_cell(st, m, F, cell);
#pragma unroll
    for (int k = 0; k < 9; ++k) st.model_cell[9 * m + k] = (float)(cell[k] / st.position_conversion);
}

// One thread per atom: v, s += dr, x = s F^T, model positions
__global__ void __launch_bounds__(MOVE_T) k_fire_move(spk_fire_t st) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * MOVE_T + threadIdx.x;
    if (a >= st.n_atoms) return;
    const int64_t m = st.idx_m[a];
    const double* c = st.coef + COEF_N * m;
    const int mode = (int)c[C_MODE];
    if (mode == MODE_FROZEN) return;
    double s[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int64_t e = 3 * a + k;
        const double v = new_velocity(c, mode, st.v[e], st.g[e]);
        st.v[e] = v;
        s[k] = st.s[e] + displacement(st, c, v);
        st.s[e] = s[k];
    }
    double x[3] = {s[0], s[1], s[2]};
    if (st.filter) {
        double F[9];
        load_F(st, m, F);
#pragma unroll
        for (int j = 0; j < 3; ++j) x[j] = dot3_rn(s[0], s[1], s[2], F[3 * j], F[3 * j + 1], F[3 * j + 2]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        st.r[3 * a + k] = x[k];
        st.model_positions[3 * a + k] = (float)(x[k] / st.position_conversion);
    }
}

bool fire_valid(const spk_fire_t* st) {
    if (!st || !st->s || !st->r || !st->v || !st->g || !st->dt || !st->a || !st->nsteps || !st->started || !st->sums ||
        !st->coef || !st->workspace || !st->counter || !st->fmax || !st->fmax_sys || !st->converged || !st->steps ||
        !st->n_unconverged || !st->model_positions || !st->idx_m || !st->sys_ptr)
        return false;
    if (st->n_atoms < 0 || st->n_sys < 1 || st->position_conversion == 0.0) return false;
    if (st->filter && (!st->h || !st->hv || !st->hg || !st->cell0 || !st->cell_factor || !st->model_cell)) return false;
    return true;
}

}  // namespace

extern "C" size_t spk_fire_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    const int64_t nb = n_atoms > 0 ? spk_cdiv(n_atoms, FIRE_T) : 0;
    return sizeof(double) * (size_t)(NSUM * ((n_sys > 0 ? n_sys : 0) + nb));
}

extern "C" int spk_fire_forces(const spk_fire_t* st, const float* forces, const double* virial, spk_stream_t stream) {
    if (!fire_valid(st) || (st->n_atoms > 0 && !forces) || (st->filter && !virial)) return SPK_ERR_ARG;
    const cudaStream_t s = spk_st(stream);
    if (st->n_atoms > 0) {
        spk_launch(k_fire_atoms, (unsigned)spk_cdiv(st->n_atoms, FIRE_T), FIRE_T, 0, s, *st, forces);
        SPK_LAUNCH_CHECK();
    }
    spk_launch(k_fire_system, (unsigned)st->n_sys, SEG_FIN_T, 0, s, *st, virial);
    SPK_LAUNCH_CHECK();
    spk_launch(k_count_unconverged<spk_fire_t>, 1, 256, 0, s, *st);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_fire_step(const spk_fire_t* st, spk_stream_t stream) {
    if (!fire_valid(st)) return SPK_ERR_ARG;
    const cudaStream_t s = spk_st(stream);
    spk_launch(k_fire_coef, (unsigned)spk_cdiv(st->n_sys, COEF_T), COEF_T, 0, s, *st);
    SPK_LAUNCH_CHECK();
    if (st->n_atoms > 0) {
        spk_launch(k_fire_move, (unsigned)spk_cdiv(st->n_atoms, MOVE_T), MOVE_T, 0, s, *st);
        SPK_LAUNCH_CHECK();
    }
    return SPK_OK;
}

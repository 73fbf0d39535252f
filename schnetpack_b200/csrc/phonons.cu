// Phonons of crystals from supercell force constants (the method of ASE's Phonons; Parlinski, Li & Kawazoe, PRL 78, 4063
// (1997)): symmetrisation and the acoustic sum rule of the force constants, the minimum-image table of the supercell,
// dynamical matrices at any q, the Gaussian density of states and the harmonic thermodynamics.
//
// Layout.  System m has n_m primitive atoms [prim_ptr[m], prim_ptr[m+1]) and a supercell of L = det(M) primitive cells
// whose atom j = l n_m + b is primitive atom b translated by lattice[l] (lattice[0] = 0).  The force constants of system m
// are the n_m * n_m L blocks Phi(a, 0; j) [3, 3] at rows fc_ptr[m] + a n_m L + j; the minimum-image table has one entry
// per row.  The finite differences come from spk_vib_assemble with n_displaced = n_m: h_raw holds, per system, the rows
// d = 3 a + alpha (displaced coordinate) of 3 n_m L columns, at 9 fc_ptr[m].
//
// Every value is written once, by one thread, in a fixed order: no atomics, bitwise reproducible.  The per-system sums
// of the thermodynamics go through the segmented pass of segscan.cuh.
#include "segscan.cuh"

namespace {

constexpr int PF_T = 256;       // force-constant elements / rows per CTA
constexpr int PI_T = 128;       // minimum-image rows per CTA
constexpr int PD_T = 128;       // dynamical-matrix elements per CTA
constexpr int PS_T = 128;       // DOS grid points per CTA
constexpr int PT_T = 256;       // thermodynamics items per CTA (segscan partials)
constexpr int PT_NV = 6;        // zero-point energy, F, S, C_v, excluded modes, imaginary modes
constexpr int MAX_Y = 65535;

// the segment s of item i for ascending ptr[0..n] (ptr[s] <= i < ptr[s + 1])
template <typename I>
__device__ __forceinline__ int64_t find_segment(const I* __restrict__ ptr, int64_t n, int64_t i) {
    int64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if ((int64_t)ptr[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

struct Row {       // force-constant row -> (system, primitive atom a, supercell atom j = l n + b)
    int64_t m, n, a, j, l, b;
};

__device__ __forceinline__ Row split_row(const spk_ph_t& p, int64_t row) {
    Row r;
    r.m = find_segment(p.fc_ptr, p.n_sys, row);
    r.n = p.prim_ptr[r.m + 1] - p.prim_ptr[r.m];
    const int64_t nl = r.n * p.n_cells, local = row - p.fc_ptr[r.m];
    r.a = local / nl;
    r.j = local - r.a * nl;
    r.l = r.j / r.n;
    r.b = r.j - r.l * r.n;
    return r;
}

// h_raw (row 3 a + alpha, column 3 j + beta per system) -> the block layout
__global__ void __launch_bounds__(PF_T) k_ph_gather(spk_ph_t p, double* __restrict__ dst) {
    SPK_PDL_ENTER();
    const int64_t e = (int64_t)blockIdx.x * PF_T + threadIdx.x;
    if (e >= 9 * p.fc_ptr[p.n_sys]) return;
    const int64_t row = e / 9, ab = e - 9 * row, al = ab / 3, be = ab - 3 * al;
    const Row r = split_row(p, row);
    const int64_t n3l = 3 * r.n * p.n_cells;
    dst[e] = p.h_raw[9 * p.fc_ptr[r.m] + (3 * r.a + al) * n3l + 3 * r.j + be];
}

// One round of ASE's Phonons.read: Phi(a, 0; b, l) <- (Phi(a, 0; b, l) + Phi(b, 0; a, -l)^T) / 2 (symmetrize), then the
// on-site block Phi(a, 0; a, 0) -= sum_j Phi(a, 0; j) over the symmetrised row (acoustic).  One thread per (a, alpha,
// beta) owns the row's elements [alpha, beta], so the row sum reads only values the thread wrote itself.
__global__ void __launch_bounds__(PF_T) k_ph_round(spk_ph_t p, const double* __restrict__ src, double* __restrict__ dst) {
    SPK_PDL_ENTER();
    const int64_t t = (int64_t)blockIdx.x * PF_T + threadIdx.x;
    const int64_t n_prim = p.prim_ptr[p.n_sys];
    if (t >= 9 * n_prim) return;
    const int64_t i = t / 9, ab = t - 9 * i, al = ab / 3, be = ab - 3 * al;
    const int64_t m = find_segment(p.prim_ptr, p.n_sys, i);
    const int64_t n = p.prim_ptr[m + 1] - p.prim_ptr[m], a = i - p.prim_ptr[m], nl = n * p.n_cells;
    const int64_t base = p.fc_ptr[m];
    double sum = 0.0;
    for (int64_t j = 0; j < nl; ++j) {
        const int64_t l = j / n, b = j - l * n;
        const double v = 0.5 * (src[9 * (base + a * nl + j) + 3 * al + be] +
                                src[9 * (base + b * nl + (int64_t)p.neg[l] * n + a) + 3 * be + al]);
        dst[9 * (base + a * nl + j) + 3 * al + be] = v;
        sum += v;
    }
    if (p.acoustic) dst[9 * (base + a * nl + a) + 3 * al + be] -= sum;
}

// The supercell-lattice images of atom j closest to atom a.  r0 = x_b + lattice[l] . cell - x_a is first wrapped to
// supercell fractional coordinates in [-1/2, 1/2] (|r0w| is then an upper bound of the shortest distance); an image S
// (integer, supercell units) at |r| <= |r0w| + tol has |f_k + S_k| height_k <= |r| for every axis k, with |f_k| <= 1/2,
// so |S_k| <= (|r0w| + tol) / height_k + 1/2 bounds the search for any skew.  Images within tol of the shortest distance
// are ties; each gets weight 1 / count.  img_lattice holds their primitive translations lattice[l] + (S - g) M.
__global__ void __launch_bounds__(PI_T) k_ph_images(spk_ph_t p) {
    SPK_PDL_ENTER();
    const int64_t row = (int64_t)blockIdx.x * PI_T + threadIdx.x;
    if (row >= p.fc_ptr[p.n_sys]) return;
    const Row r = split_row(p, row);
    const double* A = p.cell + 9 * r.m;
    const double* C = p.super_cell + 9 * r.m;
    const double* Ci = p.super_inv + 9 * r.m;
    const double* xa = p.positions + 3 * (p.prim_ptr[r.m] + r.a);
    const double* xb = p.positions + 3 * (p.prim_ptr[r.m] + r.b);
    const int* nl = p.lattice + 3 * r.l;
    double r0[3], f[3];
    int g[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
        r0[k] = xb[k] + (double)nl[0] * A[k] + (double)nl[1] * A[3 + k] + (double)nl[2] * A[6 + k] - xa[k];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        f[i] = r0[0] * Ci[i] + r0[1] * Ci[3 + i] + r0[2] * Ci[6 + i];
        g[i] = (int)rint(f[i]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) r0[k] -= (double)g[0] * C[k] + (double)g[1] * C[3 + k] + (double)g[2] * C[6 + k];
    const double len = sqrt(r0[0] * r0[0] + r0[1] * r0[1] + r0[2] * r0[2]);
    int K[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) K[i] = (int)floor((len + p.tie_tol) / p.heights[3 * r.m + i] + 0.5);
    double best = len;
    for (int s0 = -K[0]; s0 <= K[0]; ++s0)
        for (int s1 = -K[1]; s1 <= K[1]; ++s1)
            for (int s2 = -K[2]; s2 <= K[2]; ++s2) {
                double d2 = 0.0;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const double x = r0[k] + s0 * C[k] + s1 * C[3 + k] + s2 * C[6 + k];
                    d2 += x * x;
                }
                best = fmin(best, sqrt(d2));
            }
    int count = 0;
    int* out = p.img_lattice + row * SPK_PH_MAX_IMAGES * 3;
    for (int s0 = -K[0]; s0 <= K[0]; ++s0)
        for (int s1 = -K[1]; s1 <= K[1]; ++s1)
            for (int s2 = -K[2]; s2 <= K[2]; ++s2) {
                double d2 = 0.0;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const double x = r0[k] + s0 * C[k] + s1 * C[3 + k] + s2 * C[6 + k];
                    d2 += x * x;
                }
                if (sqrt(d2) > best + p.tie_tol) continue;
                if (count < SPK_PH_MAX_IMAGES) {
                    const int S[3] = {s0 - g[0], s1 - g[1], s2 - g[2]};
#pragma unroll
                    for (int k = 0; k < 3; ++k)
                        out[3 * count + k] = nl[k] + S[0] * p.supercell[k] + S[1] * p.supercell[3 + k] +
                                             S[2] * p.supercell[6 + k];
                }
                ++count;
            }
    p.img_count[row] = count;
}

// D_{a alpha, b beta}(q) = sum_l sum_images w Phi(a, 0; l n + b)[alpha, beta] e^{2 pi i q . n_image} mw / sqrt(m_a m_b)
__global__ void __launch_bounds__(PD_T) k_ph_dynmat(spk_ph_t p, const double* __restrict__ q, int64_t n_q,
                                                    const int64_t* __restrict__ dyn_ptr, double2* __restrict__ dyn) {
    SPK_PDL_ENTER();
    const int64_t e = (int64_t)blockIdx.x * PD_T + threadIdx.x;
    const int64_t n_el = dyn_ptr[p.n_sys];
    if (e >= n_el) return;
    const int64_t m = find_segment(dyn_ptr, p.n_sys, e);
    const int64_t first = p.prim_ptr[m], n = p.prim_ptr[m + 1] - first, n3 = 3 * n, nl = n * p.n_cells;
    const int64_t local = e - dyn_ptr[m], rr = local / n3, cc = local - rr * n3;
    const int64_t a = rr / 3, al = rr - 3 * a, b = cc / 3, be = cc - 3 * b;
    const double scale = p.mw_scale / sqrt(p.masses[first + a] * p.masses[first + b]);
    for (int64_t iq = blockIdx.y; iq < n_q; iq += gridDim.y) {
        const double q0 = q[3 * iq], q1 = q[3 * iq + 1], q2 = q[3 * iq + 2];
        double re = 0.0, im = 0.0;
        for (int64_t l = 0; l < p.n_cells; ++l) {
            const int64_t row = p.fc_ptr[m] + a * nl + l * n + b;
            const double phi = p.force_constants[9 * row + 3 * al + be];
            const int cnt = p.img_count[row];
            const int* img = p.img_lattice + row * SPK_PH_MAX_IMAGES * 3;
            double c = 0.0, s = 0.0;
            for (int k = 0; k < cnt; ++k) {
                double sk, ck;
                sincospi(2.0 * (q0 * img[3 * k] + q1 * img[3 * k + 1] + q2 * img[3 * k + 2]), &sk, &ck);
                c += ck;
                s += sk;
            }
            re += phi * c / cnt;
            im += phi * s / cnt;
        }
        dyn[iq * n_el + e] = make_double2(re * scale, im * scale);
    }
}

// g(E) = sum_q sum_k exp(-(E - w)^2 / (2 width^2)) / (width sqrt(2 pi) n_q) over the 3 n_m modes of system m
__global__ void __launch_bounds__(PS_T) k_ph_dos(const double* __restrict__ freq, int64_t n_q, int64_t n_modes,
                                                 const int32_t* __restrict__ prim_ptr, const double* __restrict__ grid,
                                                 int64_t n_grid, double width, double* __restrict__ out) {
    SPK_PDL_ENTER();
    const int64_t gi = (int64_t)blockIdx.x * PS_T + threadIdx.x;
    const int64_t m = blockIdx.y;
    if (gi >= n_grid) return;
    const int64_t lo = 3 * (int64_t)prim_ptr[m], k3 = 3 * (int64_t)prim_ptr[m + 1] - lo;
    const double E = grid[gi], inv_w = 1.0 / width;
    double acc = 0.0;
    for (int64_t iq = 0; iq < n_q; ++iq)
        for (int64_t k = 0; k < k3; ++k) {
            const double u = (E - freq[iq * n_modes + lo + k]) * inv_w;
            acc += exp(-0.5 * u * u);
        }
    out[m * n_grid + gi] = acc * inv_w * 0.3989422804014327 / (double)n_q;      // 1 / sqrt(2 pi)
}

// ln(1 - e^-x) for x > 0 without cancellation at either end
__device__ __forceinline__ double log1mexp(double x) {
    return x > 0.6931471805599453 ? log1p(-exp(-x)) : log(-expm1(-x));
}

// Items of segment s = (temperature t, system m), s = t B + m, are the (q, k) modes of system m; each contributes
// hbar w / 2, hbar w / 2 + kT ln(1 - e^-x), k_B (x / (e^x - 1) - ln(1 - e^-x)) and k_B (x / (2 sinh(x / 2)))^2 with
// x = hbar w / kT (T = 0: the zero-point terms only), divided by n_q; modes below min_freq are left out and counted.
__global__ void __launch_bounds__(PT_T) k_ph_thermo(const double* __restrict__ freq, int64_t n_q, int64_t n_modes,
                                                    const int32_t* __restrict__ prim_ptr, int64_t n_sys,
                                                    const double* __restrict__ temperatures,
                                                    const int32_t* __restrict__ seg_ptr, int64_t n_seg,
                                                    double min_freq, double ev_per_invcm, double k_b,
                                                    double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t i = (int64_t)blockIdx.x * PT_T + threadIdx.x;
    const int64_t n_items = seg_ptr[n_seg];
    double v[PT_NV];
#pragma unroll
    for (int c = 0; c < PT_NV; ++c) v[c] = 0.0;
    int64_t s = 0, first = 0, end = 0;
    if (i < n_items) {
        s = find_segment(seg_ptr, n_seg, i);
        first = seg_ptr[s];
        end = seg_ptr[s + 1];
        const int64_t t = s / n_sys, m = s - t * n_sys;
        const int64_t lo = 3 * (int64_t)prim_ptr[m], k3 = 3 * (int64_t)prim_ptr[m + 1] - lo;
        const int64_t local = i - first, iq = local / k3, k = local - iq * k3;
        const double w = freq[iq * n_modes + lo + k];
        if (w < min_freq) {
            v[4] = 1.0;
            v[5] = w < 0.0 ? 1.0 : 0.0;
        } else {
            const double inv_nq = 1.0 / (double)n_q, eps = w * ev_per_invcm, kt = k_b * temperatures[t];
            v[0] = 0.5 * eps * inv_nq;
            v[1] = v[0];
            if (kt > 0.0) {
                const double x = eps / kt, lg = log1mexp(x), y = x / (2.0 * sinh(0.5 * x));
                v[1] += kt * lg * inv_nq;
                v[2] = k_b * (x / expm1(x) - lg) * inv_nq;
                v[3] = k_b * y * y * inv_nq;
            }
        }
    }
    seg_partials<PT_T, PT_NV>(v, n_items, s, first, end, sys_part, head);
}

int check_params(const spk_ph_t* p) {
    if (!p || p->n_sys < 1 || p->n_cells < 1 || !p->prim_ptr || !p->fc_ptr) return SPK_ERR_ARG;
    return SPK_OK;
}

unsigned grid_x(int64_t n, int t) { return (unsigned)(n > 0 ? spk_cdiv(n, t) : 1); }

}  // namespace

extern "C" int spk_ph_force_constants(const spk_ph_t* p, spk_stream_t stream) {
    if (check_params(p) != SPK_OK || !p->h_raw || !p->force_constants || !p->work || !p->neg || p->rounds < 0)
        return SPK_ERR_ARG;
    const int64_t rows = p->n_rows, n_prim = p->n_prim;
    // without the sum rule a second symmetrisation is the identity (exactly: (v + v) / 2 = v)
    const int64_t rounds = p->acoustic ? p->rounds : (p->rounds > 0 ? 1 : 0);
    double* cur = rounds % 2 ? p->work : p->force_constants;
    spk_launch(k_ph_gather, grid_x(9 * rows, PF_T), PF_T, 0, spk_st(stream), *p, cur);
    SPK_LAUNCH_CHECK();
    for (int64_t r = 0; r < rounds; ++r) {
        double* nxt = cur == p->work ? p->force_constants : p->work;
        spk_launch(k_ph_round, grid_x(9 * n_prim, PF_T), PF_T, 0, spk_st(stream), *p, (const double*)cur, nxt);
        SPK_LAUNCH_CHECK();
        cur = nxt;
    }
    return SPK_OK;
}

extern "C" int spk_ph_images(const spk_ph_t* p, spk_stream_t stream) {
    if (check_params(p) != SPK_OK || !p->lattice || !p->positions || !p->cell || !p->super_cell || !p->super_inv ||
        !p->heights || !p->img_count || !p->img_lattice || !(p->tie_tol >= 0.0))
        return SPK_ERR_ARG;
    spk_launch(k_ph_images, grid_x(p->n_rows, PI_T), PI_T, 0, spk_st(stream), *p);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_ph_dynmat(const spk_ph_t* p, const double* q, int64_t n_q, const int64_t* dyn_ptr, void* dyn,
                             spk_stream_t stream) {
    if (check_params(p) != SPK_OK || !p->force_constants || !p->img_count || !p->img_lattice || !p->masses || !q ||
        !dyn_ptr || !dyn || n_q < 0 || p->max_atoms < 1)
        return SPK_ERR_ARG;
    if (n_q == 0) return SPK_OK;
    // dyn_ptr[B] is on the device: size the grid from the largest system, max_atoms
    const int64_t n_el = 9 * p->max_atoms * p->max_atoms * p->n_sys;
    const dim3 grid(grid_x(n_el, PD_T), (unsigned)(n_q < MAX_Y ? n_q : MAX_Y));
    spk_launch(k_ph_dynmat, grid, PD_T, 0, spk_st(stream), *p, q, n_q, dyn_ptr, (double2*)dyn);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_ph_dos(const double* freq, int64_t n_q, int64_t n_modes, const int32_t* prim_ptr, int64_t n_sys,
                          const double* grid, int64_t n_grid, double width, double* out, spk_stream_t stream) {
    if (!freq || !prim_ptr || !grid || !out || n_q < 1 || n_modes < 0 || n_sys < 1 || n_sys > MAX_Y || n_grid < 0 ||
        !(width > 0.0))
        return SPK_ERR_ARG;
    if (n_grid == 0) return SPK_OK;
    const dim3 g(grid_x(n_grid, PS_T), (unsigned)n_sys);
    spk_launch(k_ph_dos, g, PS_T, 0, spk_st(stream), freq, n_q, n_modes, prim_ptr, grid, n_grid, width, out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" size_t spk_ph_thermo_workspace_bytes(int64_t n_items, int64_t n_seg) {
    return sizeof(double) * PT_NV * (size_t)(n_seg + spk_cdiv(n_items > 0 ? n_items : 1, PT_T));
}

extern "C" int spk_ph_thermo(const double* freq, int64_t n_q, int64_t n_modes, const int32_t* prim_ptr, int64_t n_sys,
                             const double* temperatures, int64_t n_temps, const int32_t* seg_ptr, int64_t n_items,
                             double min_freq, double ev_per_invcm, double k_b, double* out, void* workspace,
                             size_t workspace_bytes, spk_stream_t stream) {
    const int64_t n_seg = n_sys * n_temps;
    if (!freq || !prim_ptr || !temperatures || !seg_ptr || !out || !workspace || n_q < 1 || n_sys < 1 || n_temps < 1 ||
        n_items < 0 || workspace_bytes < spk_ph_thermo_workspace_bytes(n_items, n_seg))
        return SPK_ERR_ARG;
    double* sys_part = (double*)workspace;
    double* head = sys_part + PT_NV * n_seg;
    spk_launch(k_ph_thermo, grid_x(n_items, PT_T), PT_T, 0, spk_st(stream), freq, n_q, n_modes, prim_ptr, n_sys,
               temperatures, seg_ptr, n_seg, min_freq, ev_per_invcm, k_b, sys_part, head);
    SPK_LAUNCH_CHECK();
    spk_launch(k_seg_finish<PT_T, PT_NV>, (unsigned)n_seg, SEG_FIN_T, 0, spk_st(stream), seg_ptr,
               (const int32_t*)nullptr, (const double*)sys_part, (const double*)head, out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

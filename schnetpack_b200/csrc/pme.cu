// Reciprocal term of smooth particle-mesh Ewald (Essmann et al., J. Chem. Phys. 103, 8577 (1995)); the real-space and
// self terms are those of the Ewald sum (pair_energy.cu, ewald.cu).  Per system m with cell h, H = h^-1, V = |det h|, a
// mesh of n1 x n2 x n3 points and cardinal B-splines M_p of even order p:
//   Q_m(x)   = sum_i q_i prod_a M_p(u_ia - x_a  mod n_a),  u_ia = n_a s_ia,  s_i = r_i H mod 1
//   E_rec[m] = sum_{j != 0} theta_j |Q^_m(j)|^2,  theta_j = ke (2 pi / V) f_k |b(j)|^2,  f_k = exp(-k^2 / (4 alpha)) / k^2
// with k = 2 pi H j over the signed mesh frequencies j and |b|^2 = prod_a |sum_{l<p-1} M_p(l+1) e^{2 pi i j_a l / n_a}|^-2.
// The FFTs between the launches are the caller's (fp64, batched over systems): Q^ = rfftn(Q), and the potential mesh
// phi = dE_rec/dQ = irfftn(conv) with conv = 2 n1 n2 n3 theta Q^.  A Nyquist frequency j_a = n_a / 2 (even n_a) has no
// sign in a triclinic cell, so its terms are left out (theta = 0); then theta is even in j, conv is Hermitian and phi is
// the exact derivative of the energy the forward reports.
//
// Layout.  Spreading is gather-based: atoms are binned by the mesh brick (PM_B^3 points) of their first support point
// with a stable counting sort (integer counts, a scan, a fill, and a per-bin sort by atom index that makes the order
// within a bin independent of the fill's atomics); one CTA per (brick, system) owns the brick's points, one per thread,
// and walks the atoms of the bricks whose support reaches into it in brick order, then bin order.  Each mesh point thus
// adds its terms in a fixed order and the mesh is written once, without atomics or a memset.  The influence pass runs
// over (system, half-spectrum frequency) and its per-system sums (E_rec and T = sum E_j (1/k^2 + 1/(4 alpha)) k (x) k,
// for the cell gradient) go through the segmented-partial pass of segscan.cuh; the reverse gathers phi and grad phi over
// each atom's p^3 support.  Every result is bitwise the same on every call, and the launch shapes depend on n_atoms,
// n_sys and the mesh only.
#include <math.h>

#include "common.cuh"
#include "ewald_common.cuh"
#include "segscan.cuh"

namespace {

constexpr int PM_T = 128;            // items per CTA of the per-atom and per-frequency passes
constexpr int PM_B = 8;              // brick edge in mesh points
constexpr int PM_BT = PM_B * PM_B * PM_B;   // threads of a spreading CTA: one per brick point
constexpr int PM_ST = 64;            // atoms staged per round of a spreading CTA
constexpr int PM_NE = 7;             // per-system sums of the influence pass: E_rec, T xx yy zz xy xz yz

static_assert(3 * PM_ST <= PM_BT, "a spreading CTA stages one (atom, axis) pair per thread");
static_assert(PM_T == SEG_FIN_T, "the per-system passes reuse the partial layout of PM_T-item CTAs");

struct PmLayout {
    double *sys, *frac, *bmod, *esys, *fpart, *apart;
    int32_t *key, *sorted, *count, *cursor, *bin_ptr, *fptr;
};

struct PmShape {
    int64_t n1, n2, n3, h3, nb1, nb2, nb3, n_brick, n_freq, n_mesh;
};

inline PmShape pm_shape(int64_t n1, int64_t n2, int64_t n3) {
    PmShape s;
    s.n1 = n1, s.n2 = n2, s.n3 = n3, s.h3 = n3 / 2 + 1;
    s.nb1 = spk_cdiv(n1, PM_B), s.nb2 = spk_cdiv(n2, PM_B), s.nb3 = spk_cdiv(n3, PM_B);
    s.n_brick = s.nb1 * s.nb2 * s.nb3;
    s.n_freq = n1 * n2 * s.h3;
    s.n_mesh = n1 * n2 * n3;
    return s;
}

// workspace in doubles (the int32 arrays follow the fp64 ones)
inline size_t pm_doubles(int64_t N, int64_t B, const PmShape& S, PmLayout* L, double* base) {
    const int64_t nbf = spk_cdiv(B * S.n_freq, PM_T), nba = spk_cdiv(N, PM_T);
    const int64_t n_sys_rec = EW_SYS * B, n_frac = 3 * N, n_bmod = S.n1 + S.n2 + S.n3, n_esys = 8 * B;
    const int64_t n_fpart = PM_NE * (B + nbf + 1), n_apart = 9 * (B + nba + 1);
    const int64_t n_bins = B * S.n_brick;
    const int64_t n_int = 2 * N + 3 * n_bins + 1 + B + 1;
    const int64_t n_dbl = n_sys_rec + n_frac + n_bmod + n_esys + n_fpart + n_apart;
    if (L) {
        L->sys = base;
        L->frac = L->sys + n_sys_rec;
        L->bmod = L->frac + n_frac;
        L->esys = L->bmod + n_bmod;
        L->fpart = L->esys + n_esys;
        L->apart = L->fpart + n_fpart;
        int32_t* ib = reinterpret_cast<int32_t*>(L->apart + n_apart);
        L->key = ib;
        L->sorted = L->key + N;
        L->count = L->sorted + N;
        L->cursor = L->count + n_bins;
        L->bin_ptr = L->cursor + n_bins;
        L->fptr = L->bin_ptr + n_bins + 1;
    }
    return (size_t)(n_dbl + (n_int + 1) / 2);
}

// Cardinal B-spline weights of order P at the fractional offset f in [0, 1): w[l] = M_P(f + P - 1 - l), the weight of
// mesh point (floor(u) - P + 1 + l), and dw[l] = dw[l]/du (Essmann et al., eqs. 4.1 and 4.4).
template <int P>
__device__ __forceinline__ void pm_spline(double f, double (&w)[P], double (&dw)[P]) {
    w[P - 1] = 0.0;
    w[1] = f;
    w[0] = 1.0 - f;
#pragma unroll
    for (int j = 3; j < P; ++j) {
        const double div = 1.0 / (j - 1);
        w[j - 1] = div * f * w[j - 2];
#pragma unroll
        for (int k = 1; k < j - 1; ++k) w[j - k - 1] = div * ((f + k) * w[j - k - 2] + (j - k - f) * w[j - k - 1]);
        w[0] = div * (1.0 - f) * w[0];
    }
    dw[0] = -w[0];
#pragma unroll
    for (int j = 1; j < P; ++j) dw[j] = w[j - 1] - w[j];
    const double div = 1.0 / (P - 1);
    w[P - 1] = div * f * w[P - 2];
#pragma unroll
    for (int k = 1; k < P - 1; ++k) w[P - k - 1] = div * ((f + k) * w[P - k - 2] + (P - k - f) * w[P - k - 1]);
    w[0] = div * (1.0 - f) * w[0];
}

// first support point (floor(u) - P + 1 mod n) and fractional offset of u = n s along one axis
template <int P>
__device__ __forceinline__ int pm_base(double s, int64_t n, double& f) {
    const double u = s * (double)n;
    const double fl = floor(u);
    f = u - fl;
    int b = (int)fl - (P - 1);
    b %= (int)n;
    return b < 0 ? b + (int)n : b;
}

// Zeroes the bin counters, writes the B-spline moduli |sum_l M_P(l+1) e^{2 pi i j l / n}|^2 of the three axes and the
// per-system frequency ranges fptr[m] = m n_freq.  Grid-stride over max(n_bins, n1 + n2 + n3, n_sys + 1) items.
template <int P>
__global__ void k_pme_setup(int64_t n_bins, int64_t n_sys, PmShape S, int32_t* __restrict__ count,
                            int32_t* __restrict__ cursor, double* __restrict__ bmod, int32_t* __restrict__ fptr) {
    SPK_PDL_ENTER();
    const int64_t n_ax = S.n1 + S.n2 + S.n3;
    const int64_t n_all = max(n_bins, max(n_ax, n_sys + 1));
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_all; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < n_bins) count[i] = 0, cursor[i] = 0;
        if (i <= n_sys) fptr[i] = (int32_t)(i * S.n_freq);
        if (i < n_ax) {
            const int64_t n = i < S.n1 ? S.n1 : (i < S.n1 + S.n2 ? S.n2 : S.n3);
            const int64_t j = i < S.n1 ? i : (i < S.n1 + S.n2 ? i - S.n1 : i - S.n1 - S.n2);
            double w[P], dw[P];
            pm_spline<P>(0.0, w, dw);                 // w[l] = M_P(P - 1 - l)
            double re = 0.0, im = 0.0;
#pragma unroll
            for (int l = 0; l < P - 1; ++l) {
                double sn, cs;
                sincospi(2.0 * (double)((j * l) % n) / (double)n, &sn, &cs);
                re = fma(w[P - 2 - l], cs, re);
                im = fma(w[P - 2 - l], sn, im);
            }
            bmod[i] = re * re + im * im;
        }
    }
}

// bin of each atom: (system, brick of its first support point); integer counts per bin
template <int P>
__global__ void k_pme_bin(const int64_t* __restrict__ idx_m, const double* __restrict__ frac, int64_t n_atoms, PmShape S,
                          int32_t* __restrict__ key, int32_t* __restrict__ count) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    double f;
    const int b1 = pm_base<P>(frac[3 * a], S.n1, f) / PM_B;
    const int b2 = pm_base<P>(frac[3 * a + 1], S.n2, f) / PM_B;
    const int b3 = pm_base<P>(frac[3 * a + 2], S.n3, f) / PM_B;
    const int32_t k = (int32_t)(idx_m[a] * S.n_brick + (b1 * S.nb2 + b2) * S.nb3 + b3);
    key[a] = k;
    atomicAdd(&count[k], 1);
}

// exclusive scan of the bin counts by one CTA of 1024 threads, each owning a contiguous run of bins
__global__ void __launch_bounds__(1024) k_pme_scan(const int32_t* __restrict__ count, int64_t n_bins,
                                                   int32_t* __restrict__ bin_ptr) {
    __shared__ int32_t tot[1024];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t per = (n_bins + 1023) / 1024;
    const int64_t b0 = min(n_bins, t * per), b1 = min(n_bins, b0 + per);
    int32_t s = 0;
    for (int64_t b = b0; b < b1; ++b) s += count[b];
    tot[t] = s;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
        const int32_t v = t >= d ? tot[t - d] : 0;
        __syncthreads();
        tot[t] += v;
        __syncthreads();
    }
    int32_t run = tot[t] - s;
    for (int64_t b = b0; b < b1; ++b) {
        bin_ptr[b] = run;
        run += count[b];
    }
    if (t == 1023) bin_ptr[n_bins] = tot[1023];
}

__global__ void k_pme_fill(const int32_t* __restrict__ key, int64_t n_atoms, const int32_t* __restrict__ bin_ptr,
                           int32_t* __restrict__ cursor, int32_t* __restrict__ sorted) {
    SPK_PDL_ENTER();
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    const int32_t k = key[a];
    sorted[bin_ptr[k] + atomicAdd(&cursor[k], 1)] = (int32_t)a;
}

// one thread per bin: insertion sort of the bin's atoms by index (a bin holds the atoms of PM_B^3 mesh points, a few
// dozen at the spacings that reach 1e-5 in condensed phase)
__global__ void k_pme_sort_bins(const int32_t* __restrict__ bin_ptr, int64_t n_bins, int32_t* __restrict__ sorted) {
    SPK_PDL_ENTER();
    const int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (b >= n_bins) return;
    const int32_t lo = bin_ptr[b], hi = bin_ptr[b + 1];
    for (int32_t i = lo + 1; i < hi; ++i) {
        const int32_t v = sorted[i];
        int32_t j = i - 1;
        while (j >= lo && sorted[j] > v) {
            sorted[j + 1] = sorted[j];
            --j;
        }
        sorted[j + 1] = v;
    }
}

// the bricks along one axis whose atoms can reach the points [x0, x1): first support points in the cyclic range
// [x0 - P + 1, x1 - 1], walked from its first brick
template <int P>
__device__ __forceinline__ void pm_brick_range(int64_t x0, int64_t x1, int64_t n, int64_t nb, int& first, int& cnt) {
    const int64_t len = x1 - x0 + P - 1;
    if (len >= n) {
        first = 0, cnt = (int)nb;
        return;
    }
    const int64_t lo = ((x0 - (P - 1)) % n + n) % n, hi = (lo + len - 1) % n;
    first = (int)(lo / PM_B);
    const int last = (int)(hi / PM_B);
    cnt = (last - first + (int)nb) % (int)nb + 1;
    if (cnt == 1 && hi < lo) cnt = (int)nb;         // wraps round to the brick it started in
}

// Q_m on the points of brick blockIdx.x of system blockIdx.y, one point per thread.  Work per CTA: PM_BT x the atoms of
// up to (1 + ceil((P - 1) / PM_B))^3 = 8 bricks (more only on meshes with a partial last brick).
template <int P>
__global__ void __launch_bounds__(PM_BT, 1) k_pme_spread(const float* __restrict__ q, const double* __restrict__ frac,
                                                      const int32_t* __restrict__ sorted,
                                                      const int32_t* __restrict__ bin_ptr, PmShape S,
                                                      double* __restrict__ mesh) {
    __shared__ int sb[3][PM_ST];
    __shared__ double sw[3][P][PM_ST];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t m = blockIdx.y;
    const int64_t br = blockIdx.x;
    const int64_t g1 = br / (S.nb2 * S.nb3), g2 = (br / S.nb3) % S.nb2, g3 = br % S.nb3;
    const int64_t x = g1 * PM_B + (t >> 6), y = g2 * PM_B + ((t >> 3) & 7), z = g3 * PM_B + (t & 7);
    int f1, c1, f2, c2, f3, c3;
    pm_brick_range<P>(g1 * PM_B, min(S.n1, (g1 + 1) * PM_B), S.n1, S.nb1, f1, c1);
    pm_brick_range<P>(g2 * PM_B, min(S.n2, (g2 + 1) * PM_B), S.n2, S.nb2, f2, c2);
    pm_brick_range<P>(g3 * PM_B, min(S.n3, (g3 + 1) * PM_B), S.n3, S.nb3, f3, c3);
    double acc = 0.0;
    for (int i1 = 0; i1 < c1; ++i1) {
        const int64_t h1 = (f1 + i1) % S.nb1;
        for (int i2 = 0; i2 < c2; ++i2) {
            const int64_t h2 = (f2 + i2) % S.nb2;
            for (int i3 = 0; i3 < c3; ++i3) {
                const int64_t bin = m * S.n_brick + (h1 * S.nb2 + h2) * S.nb3 + (f3 + i3) % S.nb3;
                const int32_t lo = bin_ptr[bin], hi = bin_ptr[bin + 1];
                for (int32_t base = lo; base < hi; base += PM_ST) {
                    const int cnt = min(PM_ST, hi - base);
                    __syncthreads();
                    if (t < 3 * PM_ST && t % PM_ST < cnt) {   // one (atom, axis) pair per thread
                        const int c = t / PM_ST, j = t % PM_ST;
                        const int64_t a = sorted[base + j];
                        double f, w[P], dw[P];
                        sb[c][j] = pm_base<P>(frac[3 * a + c], c == 0 ? S.n1 : (c == 1 ? S.n2 : S.n3), f);
                        pm_spline<P>(f, w, dw);
                        const double sc = c == 0 ? (double)q[a] : 1.0;
#pragma unroll
                        for (int l = 0; l < P; ++l) sw[c][l][j] = sc * w[l];
                    }
                    __syncthreads();
                    for (int j = 0; j < cnt; ++j) {
                        int64_t d1 = x - sb[0][j], d2 = y - sb[1][j], d3 = z - sb[2][j];
                        if (d1 < 0) d1 += S.n1;
                        if (d2 < 0) d2 += S.n2;
                        if (d3 < 0) d3 += S.n3;
                        if (d1 < P && d2 < P && d3 < P) acc += sw[0][d1][j] * sw[1][d2][j] * sw[2][d3][j];
                    }
                }
            }
        }
    }
    if (x < S.n1 && y < S.n2 && z < S.n3) mesh[((m * S.n1 + x) * S.n2 + y) * S.n3 + z] = acc;
}

// One thread per (system, half-spectrum frequency): theta, the energy term E_j = w_j theta |Q^|^2 (w_j = 2 for the
// frequencies the half spectrum stands for twice), conv = 2 n1 n2 n3 theta Q^, and the partials of E_rec and T.
__global__ void __launch_bounds__(PM_T) k_pme_influence(const double* __restrict__ sys, const double* __restrict__ bmod,
                                                        const double2* __restrict__ spec, int64_t n_sys, PmShape S,
                                                        double ke, double alpha, double2* __restrict__ conv,
                                                        double* __restrict__ fpart, double* __restrict__ fhead) {
    SPK_PDL_ENTER();
    const int64_t n_items = n_sys * S.n_freq;
    const int64_t i = (int64_t)blockIdx.x * PM_T + threadIdx.x;
    double v[PM_NE];
#pragma unroll
    for (int c = 0; c < PM_NE; ++c) v[c] = 0.0;
    int64_t m = 0, first = 0, end = 0;
    if (i < n_items) {
        m = i / S.n_freq;
        first = m * S.n_freq, end = first + S.n_freq;
        const int64_t r = i - first;
        const int64_t j1 = r / (S.n2 * S.h3), j2 = (r / S.h3) % S.n2, j3 = r % S.h3;
        const bool nyq = (2 * j1 == S.n1) || (2 * j2 == S.n2) || (2 * j3 == S.n3);
        const double m1 = (double)(2 * j1 < S.n1 ? j1 : j1 - S.n1), m2 = (double)(2 * j2 < S.n2 ? j2 : j2 - S.n2);
        const double m3 = (double)j3;
        const double* H = sys + EW_SYS * m;
        const double kx = 2.0 * EW_PI * (m1 * H[0] + m2 * H[1] + m3 * H[2]);
        const double ky = 2.0 * EW_PI * (m1 * H[3] + m2 * H[4] + m3 * H[5]);
        const double kz = 2.0 * EW_PI * (m1 * H[6] + m2 * H[7] + m3 * H[8]);
        const double k2 = kx * kx + ky * ky + kz * kz;
        double theta = 0.0;
        if (!nyq && (j1 | j2 | j3) != 0) {
            const double b = bmod[j1] * bmod[S.n1 + j2] * bmod[S.n1 + S.n2 + j3];
            theta = ke * 2.0 * EW_PI / H[9] * exp(-0.25 * k2 / alpha) / k2 / b;
        }
        const double2 Q = spec[i];
        const double sc = 2.0 * (double)S.n_mesh * theta;
        conv[i] = make_double2(sc * Q.x, sc * Q.y);
        if (theta != 0.0) {
            const double e = (j3 == 0 ? 1.0 : 2.0) * theta * (Q.x * Q.x + Q.y * Q.y);
            const double w = e * (1.0 / k2 + 0.25 / alpha);
            v[0] = e;
            v[1] = w * kx * kx, v[2] = w * ky * ky, v[3] = w * kz * kz;
            v[4] = w * kx * ky, v[5] = w * kx * kz, v[6] = w * ky * kz;
        }
    }
    seg_partials<PM_T, PM_NE>(v, n_items, m, first, end, fpart, fhead);
}

// energy[m] = addend[m] + E_rec - ke sqrt(alpha / pi) sum_i q_i^2; E_rec and T kept for the reverse
__global__ void __launch_bounds__(SEG_FIN_T) k_pme_energy(const float* __restrict__ q, const int32_t* __restrict__ sys_ptr,
                                                          const int32_t* __restrict__ fptr, const double* __restrict__ sys,
                                                          const double* __restrict__ fpart,
                                                          const double* __restrict__ fhead, double ke, double alpha,
                                                          const float* __restrict__ addend, float* __restrict__ energy,
                                                          double* __restrict__ esys) {
    __shared__ double red[PM_NE][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t m = blockIdx.x;
    seg_finish_block<PM_T, PM_NE>(fptr, nullptr, fpart, fhead, m, red);
    double tot[PM_NE];
#pragma unroll
    for (int c = 0; c < PM_NE; ++c) tot[c] = red[c][0];
    __syncthreads();
    double acc[1] = {0.0};
    for (int64_t a = sys_ptr[m] + t; a < sys_ptr[m + 1]; a += SEG_FIN_T) acc[0] += (double)q[a] * (double)q[a];
    ew_tree<1>(acc, red);
    if (t != 0) return;
#pragma unroll
    for (int c = 0; c < PM_NE; ++c) esys[8 * m + c] = tot[c];
    const double V = sys[EW_SYS * m + 9];
    double e = tot[0] - ke * sqrt(alpha / EW_PI) * red[0][0];
    if (!(V > 0.0)) e = __longlong_as_double(0x7ff8000000000000ll);     // zero volume: the reference raises
    energy[m] = (float)((addend ? (double)addend[m] : 0.0) + e);
}

// Per atom: phi_i and grad_u phi_i over the P^3 support, then g_R, g_q and the partials of sum_i r_i (x) g_R_i
template <int P>
__global__ void __launch_bounds__(PM_T) k_pme_gather(const float* __restrict__ R, const float* __restrict__ q,
                                                     const int64_t* __restrict__ idx_m,
                                                     const int32_t* __restrict__ sys_ptr,
                                                     const double* __restrict__ sys, const double* __restrict__ frac,
                                                     const double* __restrict__ phi, int64_t n_atoms, PmShape S,
                                                     double ke, double alpha, const float* __restrict__ g_E,
                                                     float* __restrict__ g_R, float* __restrict__ g_q, int accumulate_q,
                                                     double* __restrict__ sys_part, double* __restrict__ head) {
    __shared__ double sw1[P][PM_T], sd1[P][PM_T];     // the first axis' weights, indexed by the rolled outer loop
    SPK_PDL_ENTER();
    const int t = threadIdx.x;
    const int64_t a = (int64_t)blockIdx.x * PM_T + t;
    double v[9];
#pragma unroll
    for (int c = 0; c < 9; ++c) v[c] = 0.0;
    int64_t m = 0, first = 0, end = 0;
    if (a < n_atoms) {
        m = idx_m[a];
        first = sys_ptr[m];
        end = sys_ptr[m + 1];
        double f, w1[P], d1[P], w2[P], d2[P], w3[P], d3[P];
        const int b1 = pm_base<P>(frac[3 * a], S.n1, f);
        pm_spline<P>(f, w1, d1);
#pragma unroll
        for (int l = 0; l < P; ++l) sw1[l][t] = w1[l], sd1[l][t] = d1[l];
        const int b2 = pm_base<P>(frac[3 * a + 1], S.n2, f);
        pm_spline<P>(f, w2, d2);
        const int b3 = pm_base<P>(frac[3 * a + 2], S.n3, f);
        pm_spline<P>(f, w3, d3);
        const double* pm = phi + m * S.n_mesh;
        double p = 0.0, g1 = 0.0, g2 = 0.0, g3 = 0.0;
#pragma unroll 1
        for (int l1 = 0; l1 < P; ++l1) {
            int64_t x = b1 + l1;
            if (x >= S.n1) x -= S.n1;
            double s = 0.0, s1 = 0.0, s2 = 0.0;       // sums over l2, l3 of w2 w3 phi, w2 d3 phi, d2 w3 phi
#pragma unroll
            for (int l2 = 0; l2 < P; ++l2) {
                int64_t y = b2 + l2;
                if (y >= S.n2) y -= S.n2;
                const double* row = pm + (x * S.n2 + y) * S.n3;
                double r = 0.0, rd = 0.0;
#pragma unroll
                for (int l3 = 0; l3 < P; ++l3) {
                    int64_t z = b3 + l3;
                    if (z >= S.n3) z -= S.n3;
                    const double ph = row[z];
                    r = fma(w3[l3], ph, r);
                    rd = fma(d3[l3], ph, rd);
                }
                s = fma(w2[l2], r, s);
                s1 = fma(w2[l2], rd, s1);
                s2 = fma(d2[l2], r, s2);
            }
            const double u1 = sw1[l1][t], v1 = sd1[l1][t];
            p = fma(u1, s, p);
            g1 = fma(v1, s, g1);
            g2 = fma(u1, s2, g2);
            g3 = fma(u1, s1, g3);
        }
        const double gE = g_E[m], qa = q[a];
        const double* H = sys + EW_SYS * m;
        const double gs[3] = {S.n1 * g1, S.n2 * g2, S.n3 * g3};      // dE/ds_c / q_i
        double gR[3];
#pragma unroll
        for (int b = 0; b < 3; ++b) gR[b] = gE * qa * (H[3 * b] * gs[0] + H[3 * b + 1] * gs[1] + H[3 * b + 2] * gs[2]);
        if (g_R) {
#pragma unroll
            for (int c = 0; c < 3; ++c) g_R[3 * a + c] = (float)gR[c];
        }
        if (g_q) {
            const double gq = gE * (p - 2.0 * ke * sqrt(alpha / EW_PI) * qa);
            g_q[a] = (float)((accumulate_q ? (double)g_q[a] : 0.0) + gq);
        }
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            const double r = R[3 * a + b];
#pragma unroll
            for (int c = 0; c < 3; ++c) v[3 * b + c] = r * gR[c];
        }
    }
    seg_partials<PM_T, 9>(v, n_atoms, m, first, end, sys_part, head);
}

// Per system: g_cell = -H^T [sum_i r_i (x) g_R_i - 2 g_E T + g_E E_rec I] and the virial -g_E (E_rec I - 2 T)
__global__ void __launch_bounds__(SEG_FIN_T) k_pme_sys_bwd(const int32_t* __restrict__ sys_ptr,
                                                           const double* __restrict__ sys,
                                                           const double* __restrict__ esys,
                                                           const float* __restrict__ g_E,
                                                           const double* __restrict__ sys_part,
                                                           const double* __restrict__ head, float* __restrict__ g_cell,
                                                           double* __restrict__ virial, int accumulate_virial) {
    __shared__ double red[9][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t m = blockIdx.x;
    seg_finish_block<PM_T, 9>(sys_ptr, nullptr, sys_part, head, m, red);
    if (threadIdx.x != 0) return;
    const double* H = sys + EW_SYS * m;
    const double* es = esys + 8 * m;
    const double gE = g_E[m];
    const double E = es[0];
    const double T[9] = {es[1], es[4], es[5], es[4], es[2], es[6], es[5], es[6], es[3]};
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

bool pm_order_ok(int order) { return order == 4 || order == 6 || order == 8; }

}  // namespace

extern "C" size_t spk_pme_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n1, int64_t n2, int64_t n3,
                                          int order) {
    if (n_atoms < 0 || n_sys < 0 || !pm_order_ok(order) || n1 < order || n2 < order || n3 < order) return 0;
    return sizeof(double) * pm_doubles(n_atoms, n_sys, pm_shape(n1, n2, n3), nullptr, nullptr);
}

static int pm_check(const float* q, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys,
                    int64_t n1, int64_t n2, int64_t n3, int order, double alpha, void* workspace,
                    size_t workspace_bytes) {
    if (n_atoms < 0 || n_sys < 0 || n_atoms >= (1ll << 31) - 1 || n_sys > 65535) return SPK_ERR_ARG;
    if (!pm_order_ok(order) || n1 < order || n2 < order || n3 < order || !(alpha > 0.0)) return SPK_ERR_ARG;
    const PmShape S = pm_shape(n1, n2, n3);
    if (n_sys * S.n_freq >= (1ll << 31) || n_sys * S.n_brick >= (1ll << 31) || S.n_brick > 2147483647ll)
        return SPK_ERR_ARG;
    if (n_sys == 0) return SPK_OK;
    if (!sys_ptr || !workspace || (n_atoms > 0 && !q)) return SPK_ERR_ARG;
    if (workspace_bytes < spk_pme_workspace_bytes(n_atoms, n_sys, n1, n2, n3, order)) return SPK_ERR_ARG;
    return SPK_OK;
}

template <int P>
static void pm_spread_launch(const float* R, const float* q, const float* cell, const int64_t* idx_m,
                             int64_t n_atoms, int64_t n_sys, const PmShape& S, double* mesh, const PmLayout& L,
                             cudaStream_t st) {
    const int64_t n_bins = n_sys * S.n_brick;
    const int64_t n_setup = max(n_bins, max(S.n1 + S.n2 + S.n3, n_sys + 1));
    spk_launch(k_ewald_cell, (unsigned)spk_cdiv(n_sys, 128), 128, 0, st, cell, n_sys, L.sys);
    spk_launch(k_pme_setup<P>, (unsigned)min(spk_cdiv(n_setup, 256), (int64_t)4096), 256, 0, st, n_bins, n_sys, S,
               L.count, L.cursor, L.bmod, L.fptr);
    if (n_atoms > 0) {
        spk_launch(k_ewald_frac, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, R, idx_m, L.sys, n_atoms, L.frac);
        spk_launch(k_pme_bin<P>, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, idx_m, L.frac, n_atoms, S, L.key, L.count);
    }
    spk_launch(k_pme_scan, 1, 1024, 0, st, L.count, n_bins, L.bin_ptr);
    if (n_atoms > 0) {
        spk_launch(k_pme_fill, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, L.key, n_atoms, L.bin_ptr, L.cursor,
                   L.sorted);
        spk_launch(k_pme_sort_bins, (unsigned)spk_cdiv(n_bins, 128), 128, 0, st, L.bin_ptr, n_bins, L.sorted);
    }
    spk_launch(k_pme_spread<P>, dim3((unsigned)S.n_brick, (unsigned)n_sys), PM_BT, 0, st, q, L.frac, L.sorted,
               L.bin_ptr, S, mesh);
}

extern "C" int spk_pme_spread(const float* R, const float* q, const float* cell, const int64_t* idx_m,
                              const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int64_t n1, int64_t n2,
                              int64_t n3, int order, double* mesh, void* workspace, size_t workspace_bytes,
                              spk_stream_t stream) {
    const int rc = pm_check(q, sys_ptr, n_atoms, n_sys, n1, n2, n3, order, 1.0, workspace, workspace_bytes);
    if (rc != SPK_OK || n_sys == 0) return rc;
    if (!cell || !mesh || (n_atoms > 0 && (!R || !idx_m))) return SPK_ERR_ARG;
    const PmShape S = pm_shape(n1, n2, n3);
    PmLayout L;
    pm_doubles(n_atoms, n_sys, S, &L, reinterpret_cast<double*>(workspace));
    const cudaStream_t st = spk_st(stream);
    if (order == 4) pm_spread_launch<4>(R, q, cell, idx_m, n_atoms, n_sys, S, mesh, L, st);
    else if (order == 6) pm_spread_launch<6>(R, q, cell, idx_m, n_atoms, n_sys, S, mesh, L, st);
    else pm_spread_launch<8>(R, q, cell, idx_m, n_atoms, n_sys, S, mesh, L, st);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_pme_energy(const float* q, const int32_t* sys_ptr, const double* spectrum, int64_t n_atoms,
                              int64_t n_sys, int64_t n1, int64_t n2, int64_t n3, int order, double ke, double alpha,
                              const float* addend, float* energy, double* conv, void* workspace,
                              size_t workspace_bytes, spk_stream_t stream) {
    const int rc = pm_check(q, sys_ptr, n_atoms, n_sys, n1, n2, n3, order, alpha, workspace, workspace_bytes);
    if (rc != SPK_OK || n_sys == 0) return rc;
    if (!spectrum || !energy || !conv) return SPK_ERR_ARG;
    const PmShape S = pm_shape(n1, n2, n3);
    PmLayout L;
    pm_doubles(n_atoms, n_sys, S, &L, reinterpret_cast<double*>(workspace));
    const cudaStream_t st = spk_st(stream);
    spk_launch(k_pme_influence, (unsigned)spk_cdiv(n_sys * S.n_freq, PM_T), PM_T, 0, st, L.sys, L.bmod,
               reinterpret_cast<const double2*>(spectrum), n_sys, S, ke, alpha, reinterpret_cast<double2*>(conv),
               L.fpart, L.fpart + PM_NE * n_sys);
    spk_launch(k_pme_energy, (unsigned)n_sys, SEG_FIN_T, 0, st, q, sys_ptr, L.fptr, L.sys, L.fpart,
               L.fpart + PM_NE * n_sys, ke, alpha, addend, energy, L.esys);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_pme_bwd(const float* R, const float* q, const int64_t* idx_m, const int32_t* sys_ptr,
                           const double* potential, int64_t n_atoms, int64_t n_sys, int64_t n1, int64_t n2, int64_t n3,
                           int order, double ke, double alpha, const float* g_E, float* g_R, float* g_q,
                           int accumulate_q, float* g_cell, double* virial, int accumulate_virial, void* workspace,
                           size_t workspace_bytes, spk_stream_t stream) {
    const int rc = pm_check(q, sys_ptr, n_atoms, n_sys, n1, n2, n3, order, alpha, workspace, workspace_bytes);
    if (rc != SPK_OK || n_sys == 0) return rc;
    if (!g_E || (n_atoms > 0 && (!R || !idx_m || !potential))) return SPK_ERR_ARG;
    const PmShape S = pm_shape(n1, n2, n3);
    PmLayout L;
    pm_doubles(n_atoms, n_sys, S, &L, reinterpret_cast<double*>(workspace));
    const cudaStream_t st = spk_st(stream);
    double* sys_part = L.apart;
    double* head = sys_part + 9 * n_sys;
    if (n_atoms > 0) {
        const unsigned nb = (unsigned)spk_cdiv(n_atoms, PM_T);
        if (order == 4)
            spk_launch(k_pme_gather<4>, nb, PM_T, 0, st, R, q, idx_m, sys_ptr, L.sys, L.frac, potential, n_atoms, S, ke,
                       alpha, g_E, g_R, g_q, accumulate_q, sys_part, head);
        else if (order == 6)
            spk_launch(k_pme_gather<6>, nb, PM_T, 0, st, R, q, idx_m, sys_ptr, L.sys, L.frac, potential, n_atoms, S, ke,
                       alpha, g_E, g_R, g_q, accumulate_q, sys_part, head);
        else
            spk_launch(k_pme_gather<8>, nb, PM_T, 0, st, R, q, idx_m, sys_ptr, L.sys, L.frac, potential, n_atoms, S, ke,
                       alpha, g_E, g_R, g_q, accumulate_q, sys_part, head);
    }
    if (g_cell || virial)
        spk_launch(k_pme_sys_bwd, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, L.sys, L.esys, g_E, sys_part, head, g_cell,
                   virial, accumulate_virial);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

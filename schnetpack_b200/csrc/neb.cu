// Climbing-image nudged elastic band forces on the device: the improved tangent of Henkelman & Jonsson, J. Chem. Phys.
// 113, 9978 (2000), and the climbing image of Henkelman, Uberuaga & Jonsson, J. Chem. Phys. 113, 9901 (2000), for every
// interior image of every band of a collated batch (band-major, image-major, one system per image).
//
// With D+ = R_{i+1} - R_i, D- = R_i - R_{i-1} and F the model force (0 on fixed atoms), the tangent is
// tau = alpha D+ + beta D- and the NEB force F + gamma tau; all three scalars follow from five per-image sums
// (a = D+.D+, b = D-.D-, c = D+.D-, d = F.D+, e = F.D-), so one segmented pass is enough:
//   k_neb_partials  one thread per atom: the (image, CTA) partials of the five sums (seg_partials of segscan.cuh);
//   k_neb_image     one CTA per interior image: the sums in CTA order, the tangent branch, the climbing image, gamma;
//   k_neb_assemble  one thread per atom: F_NEB = F + gamma (alpha D+ + beta D-), fp32, 0 on fixed atoms.
// Every sum has a fixed order given the layout and there are no atomics: replays are bitwise reproducible.
#include "relax_common.cuh"
#include "segscan.cuh"

namespace {

constexpr int NEB_T = 256;       // atoms per CTA of the partial and assembly passes
constexpr int NSUM = 5;          // D+.D+, D-.D-, D+.D-, F.D+, F.D-
enum { C_ALPHA = 0, C_BETA, C_GAMMA, COEF_N };
enum { G_TNORM = 0, G_FTAU, G_SPRING, G_DPLUS, G_DMINUS, G_CLIMB, DIAG_N };

__device__ __forceinline__ double* ws_img_part(const spk_neb_t& st) { return st.workspace; }
__device__ __forceinline__ double* ws_head(const spk_neb_t& st) {
    return st.workspace + NSUM * st.n_bands * st.n_images;
}

// The two differences and the scaled force of atom a of image img (band b = img / n, interior image i = img % n)
struct AtomTerms {
    double dp[3], dm[3], f[3];
};

__device__ __forceinline__ void atom_terms(const spk_neb_t& st, const float* __restrict__ forces, int64_t a, int64_t img,
                                           AtomTerms& t) {
    const int64_t n = st.n_images;
    const int64_t b = img / n, i = img - b * n;
    const int64_t p0 = st.band_ptr[b];
    const int64_t A = (st.band_ptr[b + 1] - p0) / n;
    const int64_t k = a - p0 - i * A;             // the atom's index within its image
    const int64_t e = p0 / n + k;                 // its endpoint row
    const double* x = st.r + 3 * a;
    const double* next = i == n - 1 ? st.r_final + 3 * e : x + 3 * A;
    const double* prev = i == 0 ? st.r_initial + 3 * e : x - 3 * A;
    const bool fixed = st.fixed && st.fixed[a];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        t.dp[c] = next[c] - x[c];
        t.dm[c] = x[c] - prev[c];
        t.f[c] = optimizer_force(fixed, forces, st.force_conversion, a, c);
    }
}

__global__ void __launch_bounds__(NEB_T) k_neb_partials(spk_neb_t st, const float* __restrict__ forces) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * NEB_T + threadIdx.x;
    double v[NSUM] = {0.0, 0.0, 0.0, 0.0, 0.0};
    int64_t m = 0, first = 0, end = 0;
    if (a < st.n_atoms) {
        m = st.idx_img[a];
        first = st.img_ptr[m];
        end = st.img_ptr[m + 1];
        AtomTerms t;
        atom_terms(st, forces, a, m, t);
        const double *dp = t.dp, *dm = t.dm, *f = t.f;
        v[0] = dot3_rn(dp[0], dp[1], dp[2], dp[0], dp[1], dp[2]);
        v[1] = dot3_rn(dm[0], dm[1], dm[2], dm[0], dm[1], dm[2]);
        v[2] = dot3_rn(dp[0], dp[1], dp[2], dm[0], dm[1], dm[2]);
        v[3] = dot3_rn(f[0], f[1], f[2], dp[0], dp[1], dp[2]);
        v[4] = dot3_rn(f[0], f[1], f[2], dm[0], dm[1], dm[2]);
    }
    seg_partials<NEB_T, NSUM>(v, st.n_atoms, m, first, end, ws_img_part(st), ws_head(st));
}

// V of interior image j (0-based) of band b, or of an endpoint (j = -1: initial, j = n: final), in optimizer units
__device__ __forceinline__ double image_energy(const spk_neb_t& st, const float* __restrict__ energies, int64_t b,
                                               int64_t j) {
    if (j < 0) return st.end_energies[2 * b];
    if (j >= st.n_images) return st.end_energies[2 * b + 1];
    return (double)energies[b * st.n_images + j] * st.energy_conversion;
}

// One CTA per interior image: the five sums, the tangent, the climbing image and the coefficients
__global__ void __launch_bounds__(SEG_FIN_T) k_neb_image(spk_neb_t st, const float* __restrict__ energies) {
    __shared__ double red[NSUM][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t img = blockIdx.x;
    seg_finish_block<NEB_T, NSUM>(st.img_ptr, nullptr, ws_img_part(st), ws_head(st), img, red);
    if (threadIdx.x != 0) return;
    const double a = red[0][0], b = red[1][0], c = red[2][0], d = red[3][0], e = red[4][0];
    const int64_t n = st.n_images;
    const int64_t band = img / n, i = img - band * n;
    // the climbing image: the highest interior V of the band, ties to the lowest index
    int64_t top = 0;
    double vtop = image_energy(st, energies, band, 0);
    for (int64_t j = 1; j < n; ++j) {
        const double vj = image_energy(st, energies, band, j);
        if (vj > vtop) {
            vtop = vj;
            top = j;
        }
    }
    const bool climb_on = *st.climb != 0;
    const bool climbing = climb_on && top == i;
    if (i == 0) st.climbing[band] = climb_on ? (int32_t)top : -1;
    const double vp = image_energy(st, energies, band, i - 1);
    const double v0 = image_energy(st, energies, band, i);
    const double vn = image_energy(st, energies, band, i + 1);
    double alpha, beta;
    if (vn > v0 && v0 > vp) {
        alpha = 1.0;
        beta = 0.0;
    } else if (vn < v0 && v0 < vp) {
        alpha = 0.0;
        beta = 1.0;
    } else {
        const double dmax = fmax(fabs(vn - v0), fabs(vp - v0)), dmin = fmin(fabs(vn - v0), fabs(vp - v0));
        if (vn > vp) {
            alpha = dmax;
            beta = dmin;
        } else {
            alpha = dmin;
            beta = dmax;
        }
    }
    double tau2 = alpha * alpha * a + 2.0 * alpha * beta * c + beta * beta * b;
    if (tau2 == 0.0) {             // flat stretch: the bisector of the two unit differences
        alpha = a > 0.0 ? 1.0 / sqrt(a) : 0.0;
        beta = b > 0.0 ? 1.0 / sqrt(b) : 0.0;
        tau2 = alpha * alpha * a + 2.0 * alpha * beta * c + beta * beta * b;
    }
    const double tn = sqrt(tau2);
    const double ftau = alpha * d + beta * e;                 // F . tau
    const double np = sqrt(a), nm = sqrt(b);
    const double spring = climbing ? 0.0 : st.k * (np - nm);
    double gamma = 0.0;
    if (tau2 > 0.0) gamma = climbing ? -2.0 * ftau / tau2 : -ftau / tau2 + spring / tn;
    double* cf = st.coef + COEF_N * img;
    cf[C_ALPHA] = alpha;
    cf[C_BETA] = beta;
    cf[C_GAMMA] = gamma;
    double* g = st.diag + DIAG_N * img;
    g[G_TNORM] = tn;
    g[G_FTAU] = tau2 > 0.0 ? ftau / tn : 0.0;
    g[G_SPRING] = spring;
    g[G_DPLUS] = np;
    g[G_DMINUS] = nm;
    g[G_CLIMB] = climbing ? 1.0 : 0.0;
}

__global__ void __launch_bounds__(NEB_T) k_neb_assemble(spk_neb_t st, const float* __restrict__ forces) {
    SPK_PDL_ENTER();
    const int64_t a = (int64_t)blockIdx.x * NEB_T + threadIdx.x;
    if (a >= st.n_atoms) return;
    float* out = st.neb_forces + 3 * a;
    if (st.fixed && st.fixed[a]) {
        out[0] = out[1] = out[2] = 0.0f;
        return;
    }
    const int64_t img = st.idx_img[a];
    AtomTerms t;
    atom_terms(st, forces, a, img, t);
    const double* cf = st.coef + COEF_N * img;
    const double alpha = cf[C_ALPHA], beta = cf[C_BETA], gamma = cf[C_GAMMA];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const double tau = __dadd_rn(__dmul_rn(alpha, t.dp[k]), __dmul_rn(beta, t.dm[k]));
        out[k] = (float)__dadd_rn(t.f[k], __dmul_rn(gamma, tau));
    }
}

bool neb_valid(const spk_neb_t* st) {
    if (!st || !st->r || !st->r_initial || !st->r_final || !st->end_energies || !st->climb || !st->idx_img ||
        !st->img_ptr || !st->band_ptr || !st->coef || !st->diag || !st->climbing || !st->neb_forces || !st->workspace)
        return false;
    return st->n_atoms >= 1 && st->n_images >= 1 && st->n_bands >= 1 && st->k > 0.0;
}

}  // namespace

extern "C" size_t spk_neb_workspace_bytes(int64_t n_atoms, int64_t n_images) {
    const int64_t nb = n_atoms > 0 ? spk_cdiv(n_atoms, NEB_T) : 0;
    return sizeof(double) * (size_t)(NSUM * ((n_images > 0 ? n_images : 0) + nb));
}

extern "C" int spk_neb_forces(const spk_neb_t* st, const float* forces, const float* energies, spk_stream_t stream) {
    if (!neb_valid(st) || !forces || !energies) return SPK_ERR_ARG;
    const cudaStream_t s = spk_st(stream);
    const unsigned atom_ctas = (unsigned)spk_cdiv(st->n_atoms, NEB_T);
    spk_launch(k_neb_partials, atom_ctas, NEB_T, 0, s, *st, forces);
    SPK_LAUNCH_CHECK();
    spk_launch(k_neb_image, (unsigned)(st->n_bands * st->n_images), SEG_FIN_T, 0, s, *st, energies);
    SPK_LAUNCH_CHECK();
    spk_launch(k_neb_assemble, atom_ctas, NEB_T, 0, s, *st, forces);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

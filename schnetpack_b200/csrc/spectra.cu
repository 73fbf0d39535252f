// Vibrational spectra from recorded MD series (md/data/spectra.py: PowerSpectrum, IRSpectrum, RamanSpectrum), fp64
// arithmetic on fp32 records.
//
// Series: one CTA per output field gathers the centroid (mean over the P replicas), optionally the central difference,
// the linear combination of up to three components (Raman's trace and differences), and normalises the field by its
// mean and population std.  Sums run in a fixed order (per-thread strides, then a fixed tree): bitwise reproducible.
//
// Autocorrelation: with n points only L <= n - 1 lags are needed, so they are computed directly instead of through a
// 2n-point FFT per field.  For a channel (fields F_c with weights w_f), A[k] = (1/n) sum_t G[t, t + k] with the Gram
// matrix G[t, t'] = sum_f (w_f z_f[t]) z_f[t'].  A warp owns AC_QW tiles of 16 rows x 8 columns placed at a FIXED column
// offset 8 q from the row block: tile q of row block t0 covers G[t0 + r, t0 + 8 q + c], i.e. lag 8 q + c - r.  Because
// the offset is relative to t0, the same accumulator serves every row block of the CTA's time chunk and every group of
// four fields: D += A_t0 B_t0 with mma.m16n8k4.f64 (A = w z rows, B = z columns, K = 4 fields; 3-field IR channels pad
// one).  The B fragments of row block t0 + 16 are those of tiles q + 2 of row block t0, so each row block shifts the
// registers by two tiles and loads two.  After the chunk, the diagonals of the tiles are summed in shared memory into
// per-(chunk, lag block) partials, which a second kernel sums over chunks in a fixed order.  The chunk length is fixed
// (SPK_SPECTRUM_CHUNK), not the chunk count: a channel's result does not depend on which channels share the launch.
//
// Transform: I[m] = 2 dt |sum_i a_i cos(pi m (2i+1) / (8L))| for m < 4L, the DCT-II form of the reference's |dt FFT| of
// the zero-padded, mirrored series.  m (2i+1) is reduced modulo 16L in integers and the cosine read from a quarter-wave
// table of cospi values (in shared memory when it fits), so no cosine of a large argument is ever taken.
#include "common.cuh"

namespace {

constexpr int SE_T = 256;                       // threads per field of the series kernel
constexpr int AC_W = 4;                         // warps per CTA of the autocorrelation
constexpr int AC_QW = 8;                        // 16x8 tiles per warp
constexpr int AC_TPC = AC_W * AC_QW;            // tiles per CTA: 8 AC_TPC lag columns
constexpr int AC_SPAN = 8 * AC_TPC + 24;        // lag slots of a CTA: [8 xb AC_TPC - 16, 8 (xb + 1) AC_TPC + 8)
constexpr int AC_CHUNK = SPK_SPECTRUM_CHUNK;    // time rows per CTA
constexpr int AR_T = 256;                       // lags per CTA of the chunk reduction
constexpr int TR_T = 256;                       // frequency bins per CTA of the transform
constexpr int TR_CH = 8;                        // channels per CTA of the transform (they share the cosines)
constexpr int TR_SMEM_MAX = 160 * 1024;         // largest quarter-wave table staged in shared memory
constexpr int64_t MAX_LAGS = int64_t(1) << 26;  // 16 L stays an int32 residue
static_assert(AC_CHUNK % 16 == 0, "chunk = whole row blocks");

__device__ __forceinline__ double block_sum(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int w = 0; w < SE_T / 32; ++w) s += red[w];
    return s;
}

__device__ __forceinline__ double centroid(const float* __restrict__ rec, int64_t t, int64_t P, int64_t stride,
                                           int64_t i) {
    double s = 0.0;
    for (int64_t r = 0; r < P; ++r) s += (double)rec[(t * P + r) * stride + i];
    return s / (double)P;
}

__global__ void __launch_bounds__(SE_T) k_spectrum_series(const float* __restrict__ rec, int64_t T, int64_t P,
                                                          int64_t stride, const int64_t* __restrict__ index,
                                                          const double* __restrict__ coef, int derivative,
                                                          double dt_fs, double* __restrict__ z,
                                                          double* __restrict__ mean_out, double* __restrict__ std_out) {
    SPK_PDL_ENTER();
    __shared__ double red[SE_T / 32];
    const int64_t f = blockIdx.x;
    const int64_t n = derivative ? T - 2 : T;
    double* zf = z + f * n;
    double s = 0.0;
    for (int64_t t = threadIdx.x; t < n; t += SE_T) {
        double x = 0.0;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int64_t i = index[3 * f + j];
            if (i < 0) continue;
            double d = centroid(rec, t, P, stride, i);
            if (derivative) d = (centroid(rec, t + 2, P, stride, i) - d) / (2.0 * dt_fs);
            x += coef[3 * f + j] * d;
        }
        zf[t] = x;
        s += x;
    }
    const double mean = block_sum(s, red) / (double)n;
    double q = 0.0;
    for (int64_t t = threadIdx.x; t < n; t += SE_T) {
        const double d = zf[t] - mean;
        q += d * d;
    }
    const double sd = sqrt(block_sum(q, red) / (double)n);
    for (int64_t t = threadIdx.x; t < n; t += SE_T) zf[t] = (zf[t] - mean) / sd;
    if (threadIdx.x == 0) {
        mean_out[f] = mean;
        std_out[f] = sd;
    }
}

__device__ __forceinline__ void dmma_16x8x4(double (&d)[4], double a0, double a1, double b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
                 : "d"(a0), "d"(a1), "d"(b));
}

// grid (lag block xb, time chunk, channel); part [C, n_chunks, n_xb, AC_SPAN]
__global__ void __launch_bounds__(AC_W * 32) k_spectrum_acf(const double* __restrict__ z, int64_t n,
                                                            const int64_t* __restrict__ ch_ptr,
                                                            const double* __restrict__ weight,
                                                            double* __restrict__ part) {
    SPK_PDL_ENTER();
    __shared__ double tiles[AC_TPC * 16 * 8];
    const int xb = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tg = lane & 3;
    const int64_t c = blockIdx.z, chunk = blockIdx.y;
    const int64_t fb = ch_ptr[c], fe = ch_ptr[c + 1];
    const int64_t cs = chunk * AC_CHUNK, ce = min(cs + AC_CHUNK, n);
    const int64_t col0 = 8 * (int64_t)(xb * AC_TPC + warp * AC_QW) + g;     // column of tile 0 relative to t0
    double acc[AC_QW][4];
#pragma unroll
    for (int q = 0; q < AC_QW; ++q) acc[q][0] = acc[q][1] = acc[q][2] = acc[q][3] = 0.0;
    for (int64_t f0 = fb; f0 < fe; f0 += 4) {
        const bool fv = f0 + tg < fe;
        const double* zf = z + (fv ? f0 + tg : fb) * n;
        const double wf = fv ? weight[f0 + tg] : 0.0;
        double b[AC_QW];
#pragma unroll
        for (int q = 0; q < AC_QW; ++q) {
            const int64_t t = cs + col0 + 8 * q;
            b[q] = fv && t < n ? zf[t] : 0.0;
        }
        for (int64_t t0 = cs; t0 < ce; t0 += 16) {
            const double a0 = fv && t0 + g < ce ? wf * zf[t0 + g] : 0.0;
            const double a1 = fv && t0 + g + 8 < ce ? wf * zf[t0 + g + 8] : 0.0;
#pragma unroll
            for (int q = 0; q < AC_QW; ++q) dmma_16x8x4(acc[q], a0, a1, b[q]);
#pragma unroll
            for (int q = 0; q < AC_QW - 2; ++q) b[q] = b[q + 2];
            const int64_t t = t0 + 16 + col0 + 8 * (AC_QW - 2);
            b[AC_QW - 2] = fv && t < n ? zf[t] : 0.0;
            b[AC_QW - 1] = fv && t + 8 < n ? zf[t + 8] : 0.0;
        }
    }
    // accumulator fragment: d0, d1 at (row g, cols 2 tg, 2 tg + 1), d2, d3 at row g + 8
#pragma unroll
    for (int q = 0; q < AC_QW; ++q) {
        double* tl = tiles + (warp * AC_QW + q) * 128;
        tl[g * 8 + 2 * tg] = acc[q][0];
        tl[g * 8 + 2 * tg + 1] = acc[q][1];
        tl[(g + 8) * 8 + 2 * tg] = acc[q][2];
        tl[(g + 8) * 8 + 2 * tg + 1] = acc[q][3];
    }
    __syncthreads();
    const int64_t n_xb = gridDim.x;
    double* out = part + ((c * gridDim.y + chunk) * n_xb + xb) * AC_SPAN;
    for (int s = threadIdx.x; s < AC_SPAN; s += AC_W * 32) {
        // slot s is lag k = 8 xb AC_TPC - 16 + s; row r of local tile u >> 3 holds it in column u & 7, u = s - 16 + r
        double v = 0.0;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int u = s - 16 + r;
            if (u >= 0 && u < 8 * AC_TPC) v += tiles[(u >> 3) * 128 + r * 8 + (u & 7)];
        }
        out[s] = v;
    }
}

// acf[c, k] = (1/n) sum over chunks (in order) of the (at most two) lag blocks holding lag k
__global__ void __launch_bounds__(AR_T) k_spectrum_acf_reduce(const double* __restrict__ part, int64_t n,
                                                              int64_t n_chunks, int64_t n_xb, int64_t L,
                                                              double* __restrict__ acf) {
    SPK_PDL_ENTER();
    const int64_t k = blockIdx.x * (int64_t)AR_T + threadIdx.x, c = blockIdx.y;
    if (k >= L) return;
    const int64_t hi = (k + 16) / (8 * AC_TPC);
    const int64_t lo = hi > 0 ? hi - 1 : 0;
    double s = 0.0;
    for (int64_t ch = 0; ch < n_chunks; ++ch) {
        for (int64_t xb = lo; xb <= hi && xb < n_xb; ++xb) {
            const int64_t slot = k + 16 - 8 * AC_TPC * xb;
            if (slot >= 0 && slot < AC_SPAN) s += part[((c * n_chunks + ch) * n_xb + xb) * AC_SPAN + slot];
        }
    }
    acf[c * L + k] = s / (double)n;
}

// tab[j] = cos(pi j / (8L)) for j <= 4L
__global__ void k_spectrum_cos_table(int64_t L, double* __restrict__ tab) {
    SPK_PDL_ENTER();
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j <= 4 * L) tab[j] = cospi((double)j / (double)(8 * L));
}

// cos(pi r / (8L)) for 0 <= r < 16L from the quarter-wave table
__device__ __forceinline__ double cos_residue(const double* tab, int r, int L4) {
    if (r <= L4) return tab[r];
    if (r <= 2 * L4) return -tab[2 * L4 - r];
    if (r <= 3 * L4) return -tab[r - 2 * L4];
    return tab[4 * L4 - r];
}

__global__ void __launch_bounds__(TR_T) k_spectrum_transform(const double* __restrict__ acf, int64_t C, int64_t L,
                                                             const double* __restrict__ window, double dt_fs,
                                                             const double* __restrict__ gtab, int stage,
                                                             double* __restrict__ out) {
    SPK_PDL_ENTER();
    extern __shared__ double stab[];
    const int L4 = (int)(4 * L), L16 = (int)(16 * L);
    const double* tab = gtab;
    if (stage) {
        for (int j = threadIdx.x; j <= L4; j += TR_T) stab[j] = gtab[j];
        __syncthreads();
        tab = stab;
    }
    const int64_t m = blockIdx.x * (int64_t)TR_T + threadIdx.x;
    const int64_t c0 = blockIdx.y * (int64_t)TR_CH;
    if (m >= L4) return;
    const int nc = (int)min((int64_t)TR_CH, C - c0);
    double acc[TR_CH];
#pragma unroll
    for (int j = 0; j < TR_CH; ++j) acc[j] = 0.0;
    const int step = (int)((2 * m) % L16);
    int r = (int)(m % L16);
    for (int64_t i = 0; i < L; ++i) {
        const double v = cos_residue(tab, r, L4);
        const double w = window ? window[i] : 1.0;
#pragma unroll
        for (int j = 0; j < TR_CH; ++j)
            if (j < nc) acc[j] += (acf[(c0 + j) * L + i] * w) * v;
        r += step;
        if (r >= L16) r -= L16;
    }
#pragma unroll
    for (int j = 0; j < TR_CH; ++j)
        if (j < nc) out[(c0 + j) * L4 + m] = fabs(2.0 * dt_fs * acc[j]);
}

int64_t n_chunks_of(int64_t n) { return spk_cdiv(n, AC_CHUNK); }
int64_t n_xb_of(int64_t L) { return spk_cdiv(spk_cdiv(L + 15, 8), AC_TPC); }

SpkSmemOnce transform_smem;

}  // namespace

extern "C" size_t spk_spectrum_workspace_bytes(int64_t n_channels, int64_t n, int64_t n_lags) {
    if (n_channels < 0 || n < 1 || n_lags < 1) return 0;
    const size_t part = (size_t)n_channels * n_chunks_of(n) * n_xb_of(n_lags) * AC_SPAN * sizeof(double);
    const size_t tab = (size_t)(4 * n_lags + 1) * sizeof(double);
    return part > tab ? part : tab;
}

extern "C" int spk_spectrum_series(const float* records, int64_t T, int64_t P, int64_t stride, const int64_t* index,
                                   const double* coef, int64_t F, int derivative, double dt_fs, double* z, double* mean,
                                   double* std, spk_stream_t stream) {
    const int64_t n = derivative ? T - 2 : T;
    if (n < 1 || P < 1 || stride < 1 || F < 0 || (derivative && !(dt_fs > 0.0))) return SPK_ERR_ARG;
    if (F == 0) return SPK_OK;
    if (!records || !index || !coef || !z || !mean || !std || F > 0x7fffffff) return SPK_ERR_ARG;
    spk_launch(k_spectrum_series, (unsigned)F, SE_T, 0, spk_st(stream), records, T, P, stride, index, coef, derivative,
               dt_fs, z, mean, std);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_spectrum_autocorrelation(const double* z, int64_t n, const int64_t* ch_ptr, const double* weight,
                                            int64_t n_channels, int64_t n_lags, double* acf, void* workspace,
                                            size_t workspace_bytes, spk_stream_t stream) {
    if (n_channels < 0 || n_lags < 1 || n_lags > n - 1 || n_lags > MAX_LAGS || n_channels > 65535) return SPK_ERR_ARG;
    if (n_channels == 0) return SPK_OK;
    if (!z || !ch_ptr || !weight || !acf || !workspace) return SPK_ERR_ARG;
    if (workspace_bytes < spk_spectrum_workspace_bytes(n_channels, n, n_lags)) return SPK_ERR_ARG;
    const int64_t n_chunks = n_chunks_of(n), n_xb = n_xb_of(n_lags);
    if (n_chunks > 65535) return SPK_ERR_ARG;
    double* part = reinterpret_cast<double*>(workspace);
    spk_launch(k_spectrum_acf, dim3((unsigned)n_xb, (unsigned)n_chunks, (unsigned)n_channels), AC_W * 32, 0,
               spk_st(stream), z, n, ch_ptr, weight, part);
    spk_launch(k_spectrum_acf_reduce, dim3((unsigned)spk_cdiv(n_lags, AR_T), (unsigned)n_channels), AR_T, 0,
               spk_st(stream), part, n, n_chunks, n_xb, n_lags, acf);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_spectrum_transform(const double* acf, int64_t n_channels, int64_t n_lags, const double* window,
                                      double dt_fs, double* out, void* workspace, size_t workspace_bytes,
                                      spk_stream_t stream) {
    if (n_channels < 0 || n_lags < 1 || n_lags > MAX_LAGS || !(dt_fs > 0.0)) return SPK_ERR_ARG;
    if (n_channels == 0) return SPK_OK;
    if (!acf || !out || !workspace || workspace_bytes < (size_t)(4 * n_lags + 1) * sizeof(double)) return SPK_ERR_ARG;
    const int64_t ygrid = spk_cdiv(n_channels, TR_CH);
    if (ygrid > 65535) return SPK_ERR_ARG;
    double* tab = reinterpret_cast<double*>(workspace);
    spk_launch(k_spectrum_cos_table, (unsigned)spk_cdiv(4 * n_lags + 1, 256), 256, 0, spk_st(stream), n_lags, tab);
    const size_t smem = (size_t)(4 * n_lags + 1) * sizeof(double);
    const int stage = smem <= (size_t)TR_SMEM_MAX;
    if (stage) {
        cudaError_t e = transform_smem.set(k_spectrum_transform, TR_SMEM_MAX);
        if (e != cudaSuccess) return SPK_CUDA_ERR(e);
    }
    spk_launch(k_spectrum_transform, dim3((unsigned)spk_cdiv(4 * n_lags, TR_T), (unsigned)ygrid), TR_T,
               stage ? smem : 0, spk_st(stream), acf, n_channels, n_lags, window, dt_fs, (const double*)tab, stage,
               out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

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
#include <algorithm>

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

// ---- streaming autocorrelation inside the captured MD step ----------------------------------------------------------
// A stream keeps, per field f of its F fields, the shifted values y = x - x[0] and
//   S[k] = sum_{t < n - k} y[t] y[t + k] (k < L),  Y = sum_t y[t],  head[t] = y[t] (t < L),  ring[t % R] = y[t],
// with R = L + SPK_SPECTRUM_STREAM_BLOCK.  The push (one thread per field) forms the field from the live state exactly
// as spk_md_record_velocities / spk_md_record and spk_spectrum_series would (fp32 values, fp64 centroid, central
// difference from a two-frame history per field), and the block update adds the band products of every complete block
// of SPK_SPECTRUM_STREAM_BLOCK samples: S[k] += sum_{j < BLOCK} y[b0 + j] y[b0 + j - k].  Samples are counted from the
// recorder's device step counter (frame r = counter[0] / every on the steps with (counter[0] + 1) % every == 0), so the
// host launches both kernels every step and no counter of the stream's own is needed.  A block update CTA of T threads
// owns one field and a tile of KT = T Q lags (Q lags per thread in registers; the tile is sized from L, up to 1024
// lags, so a short lag window computes no lags it throws away beyond rounding T up to a warp): it stages the block and
// the KT + BLOCK - 1 ring values it needs in shared memory and reads and writes S once per block.  Sums run in sample
// order and in fixed blocks, so the accumulators do not depend on how the run is chunked.
namespace {

constexpr int SB = SPK_SPECTRUM_STREAM_BLOCK;   // samples per block update
constexpr int SP_T = 256;                       // fields per CTA of the push
constexpr int SU_T = 256;                       // largest CTA of the block update
constexpr int SU_KT = 4 * SU_T;                 // largest lag tile of the block update (Q = 4)
constexpr int SF_T = 256;                       // threads per field of the finalisation
constexpr int SC_T = 256;                       // lags per CTA of the channel sums
constexpr int SCAL = 8;                         // per-field scalars: Y, shift, two frames of three components

struct StreamView {
    double *S, *head, *ring, *scal;
    int64_t R;
};

__host__ __device__ __forceinline__ StreamView stream_view(double* st, int64_t F, int64_t L) {
    StreamView v;
    v.R = L + SB;
    v.S = st;
    v.head = st + F * L;
    v.ring = st + 2 * F * L;
    v.scal = st + F * (2 * L + v.R);
    return v;
}

// the centroid of component i of the live state: fp32 src (divided by the fp32 masses when given, as the velocity
// recorder does), replicas summed in order in fp64 and divided by P, as spk_spectrum_series does on the records
__device__ __forceinline__ double live_centroid(const float* __restrict__ src, const float* __restrict__ masses,
                                                int64_t P, int64_t stride, int64_t i) {
    double s = 0.0;
    for (int64_t r = 0; r < P; ++r) {
        const int64_t j = r * stride + i;
        const float v = masses ? src[j] / masses[j / 3] : src[j];
        s += (double)v;
    }
    return s / (double)P;
}

__global__ void __launch_bounds__(SP_T) k_stream_push(const float* __restrict__ src, const float* __restrict__ masses,
                                                      int64_t P, int64_t stride, const int64_t* __restrict__ index,
                                                      const double* __restrict__ coef, int64_t F, int derivative,
                                                      double dt_fs, const int64_t* __restrict__ counter, int64_t every,
                                                      int64_t L, double* __restrict__ state) {
    SPK_PDL_ENTER();
    const int64_t f = blockIdx.x * (int64_t)SP_T + threadIdx.x;
    const int64_t c0 = counter[0];
    if (f >= F || (c0 + 1) % every != 0) return;
    const int64_t r = c0 / every;
    const int64_t u = derivative ? r - 2 : r;
    const StreamView v = stream_view(state, F, L);
    double* sc = v.scal + SCAL * f;
    double x = 0.0;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const int64_t i = index[3 * f + j];
        if (i < 0) continue;
        double d = live_centroid(src, masses, P, stride, i);
        if (derivative) {
            double* h = sc + 2 + 3 * (r & 1) + j;       // c(r - 2), then c(r) for frame r + 2
            const double c = d;
            d = (c - *h) / (2.0 * dt_fs);
            *h = c;
        }
        x += coef[3 * f + j] * d;
    }
    if (u < 0) return;
    if (u == 0) sc[1] = x;
    const double y = x - sc[1];
    v.ring[f * v.R + u % v.R] = y;
    if (u < L) v.head[f * L + u] = y;
    sc[0] += y;
}

// T threads (SU_T when Q > 1, else blockDim.x), Q lags each: a tile of KT = T Q lags
template <int Q>
__global__ void __launch_bounds__(SU_T) k_stream_update(int64_t F, int derivative, const int64_t* __restrict__ counter,
                                                        int64_t every, int64_t L, double* __restrict__ state) {
    SPK_PDL_ENTER();
    __shared__ double blk[SB];
    __shared__ double seg[SU_KT + SB];
    const int64_t c0 = counter[0];
    if ((c0 + 1) % every != 0) return;
    const int64_t u = c0 / every - (derivative ? 2 : 0);
    if (u < 0 || (u + 1) % SB != 0) return;
    const int64_t b0 = u + 1 - SB;
    const StreamView v = stream_view(state, F, L);
    const int T = Q > 1 ? SU_T : (int)blockDim.x, KT = T * Q, tid = (int)threadIdx.x;     // T is fixed when Q > 1
    const int64_t n_tiles = (L + KT - 1) / KT, items = F * n_tiles;
    for (int64_t it = blockIdx.x; it < items; it += gridDim.x) {
        const int64_t f = it / n_tiles, k0 = (it % n_tiles) * KT;
        const double* ring = v.ring + f * v.R;
        const int64_t base = b0 - k0 - KT + 1;       // seg[i] = y[base + i]
        __syncthreads();
        for (int i = tid; i < KT + SB - 1; i += T) {
            const int64_t t = base + i;
            seg[i] = t >= 0 ? ring[t % v.R] : 0.0;
        }
        for (int i = tid; i < SB; i += T) blk[i] = ring[(b0 + i) % v.R];
        __syncthreads();
        double acc[Q];
#pragma unroll
        for (int q = 0; q < Q; ++q) acc[q] = 0.0;
#pragma unroll 4
        for (int j = 0; j < SB; ++j) {
            const double a = blk[j];
#pragma unroll
            for (int q = 0; q < Q; ++q) acc[q] = fma(a, seg[j - tid - T * q + KT - 1], acc[q]);
        }
        double* S = v.S + f * L;
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const int64_t k = k0 + tid + T * q;
            if (k < L) S[k] += acc[q];
        }
    }
}

// C[i, k] for k < Lo of stream field fields[i] after n samples: the partial block is added to S, the head and tail
// sums come from chunked prefix sums (thread t owns lags [t per, (t + 1) per)), then
// C[k] = (S[k] - m (2 Y - H[k] - tail[k]) + (n - k) m^2) / (n var),  m = Y / n,  var = S[0] / n - m^2.
__global__ void __launch_bounds__(SF_T) k_stream_finalise(const double* __restrict__ state, int64_t F, int64_t L,
                                                          int64_t n, const int64_t* __restrict__ fields, int64_t Lo,
                                                          double* __restrict__ out) {
    SPK_PDL_ENTER();
    __shared__ double part[2][SF_T + 1];
    const int64_t i = blockIdx.x, f = fields[i];
    const StreamView v = stream_view(const_cast<double*>(state), F, L);
    const double* S = v.S + f * L;
    const double* head = v.head + f * L;
    const double* ring = v.ring + f * v.R;
    const double Y = v.scal[SCAL * f];
    const int64_t b0 = n - n % SB;
    const int64_t per = (Lo + SF_T - 1) / SF_T;
    const int64_t ka = min(Lo, threadIdx.x * per), kb = min(Lo, ka + per);
    double* o = out + i * Lo;
    double h = 0.0, tl = 0.0;
    for (int64_t k = ka; k < kb; ++k) {
        double s = S[k];
        for (int64_t t = max(b0, k); t < n; ++t) s += ring[t % v.R] * ring[(t - k) % v.R];
        o[k] = s;
        h += head[k];
        tl += ring[(n - 1 - k) % v.R];
    }
    part[0][threadIdx.x] = h;
    part[1][threadIdx.x] = tl;
    __syncthreads();
    if (threadIdx.x == 0) {
        double a = 0.0, b = 0.0;
        for (int t = 0; t < SF_T; ++t) {
            const double pa = part[0][t], pb = part[1][t];
            part[0][t] = a;
            part[1][t] = b;
            a += pa;
            b += pb;
        }
        part[0][SF_T] = o[0];
    }
    __syncthreads();
    const double dn = (double)n, m = Y / dn;
    const double var = part[0][SF_T] / dn - m * m;
    double H = part[0][threadIdx.x], T = part[1][threadIdx.x];
    for (int64_t k = ka; k < kb; ++k) {
        o[k] = (o[k] - m * (2.0 * Y - H - T) + (double)(n - k) * m * m) / (dn * var);
        H += head[k];
        T += ring[(n - 1 - k) % v.R];
    }
}

// acf[c, k] = sum_{i in [ch_ptr[c], ch_ptr[c+1])} weight[i] C[i, k], fields in order
__global__ void __launch_bounds__(SC_T) k_stream_channels(const double* __restrict__ C, int64_t Lo,
                                                          const int64_t* __restrict__ ch_ptr,
                                                          const double* __restrict__ weight, double* __restrict__ acf) {
    SPK_PDL_ENTER();
    const int64_t k = blockIdx.x * (int64_t)SC_T + threadIdx.x, c = blockIdx.y;
    if (k >= Lo) return;
    double s = 0.0;
    for (int64_t i = ch_ptr[c]; i < ch_ptr[c + 1]; ++i) s += weight[i] * C[i * Lo + k];
    acf[c * Lo + k] = s;
}

}  // namespace

extern "C" size_t spk_spectrum_stream_state_bytes(int64_t n_fields, int64_t n_lags) {
    if (n_fields < 0 || n_lags < 1) return 0;
    return sizeof(double) * (size_t)n_fields * (size_t)(3 * n_lags + SB + SCAL);
}

extern "C" size_t spk_spectrum_stream_finalise_workspace_bytes(int64_t n_fields, int64_t n_lags) {
    if (n_fields < 0 || n_lags < 1) return 0;
    return sizeof(double) * (size_t)n_fields * (size_t)n_lags;
}

extern "C" int spk_spectrum_stream_push(const float* source, const float* masses, int64_t P, int64_t stride,
                                        const int64_t* index, const double* coef, int64_t F, int derivative,
                                        double dt_fs, const int64_t* counter, int64_t every, int64_t n_lags,
                                        double* state, spk_stream_t stream) {
    if (P < 1 || stride < 1 || F < 0 || every < 1 || n_lags < 1 || n_lags > MAX_LAGS) return SPK_ERR_ARG;
    if (derivative && !(dt_fs > 0.0)) return SPK_ERR_ARG;
    if (F == 0) return SPK_OK;
    if (!source || !index || !coef || !counter || !state || (masses && stride % 3 != 0)) return SPK_ERR_ARG;
    const cudaStream_t st = spk_st(stream);
    spk_launch(k_stream_push, (unsigned)spk_cdiv(F, SP_T), SP_T, 0, st, source, masses, P, stride, index, coef, F,
               derivative, dt_fs, counter, every, n_lags, state);
    // the lag tile from L: 1024 lags (Q = 4) above 512, 512 (Q = 2) above 256, else one lag per thread of a CTA of
    // L rounded up to a warp
    const int Q = n_lags > 512 ? 4 : n_lags > 256 ? 2 : 1;
    const int T = Q > 1 ? SU_T : (int)spk_cdiv(n_lags, 32) * 32;
    const int64_t items = F * spk_cdiv(n_lags, (int64_t)T * Q);
    const int64_t grid = std::min<int64_t>(items, 8 * (int64_t)spk_num_sms());
    if (Q == 4)
        spk_launch(k_stream_update<4>, (unsigned)grid, T, 0, st, F, derivative, counter, every, n_lags, state);
    else if (Q == 2)
        spk_launch(k_stream_update<2>, (unsigned)grid, T, 0, st, F, derivative, counter, every, n_lags, state);
    else
        spk_launch(k_stream_update<1>, (unsigned)grid, T, 0, st, F, derivative, counter, every, n_lags, state);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_spectrum_stream_finalise(const double* state, int64_t F, int64_t n_lags, int64_t n,
                                            const int64_t* fields, int64_t n_sel, const int64_t* ch_ptr,
                                            const double* weight, int64_t n_channels, int64_t n_out, double* acf,
                                            void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (F < 0 || n_lags < 1 || n_sel < 0 || n_channels < 0 || n_out < 1 || n_out > n_lags || n_out > n - 1)
        return SPK_ERR_ARG;
    if (n_channels == 0) return SPK_OK;
    if (!state || !fields || !ch_ptr || !weight || !acf || !workspace || n_sel > 0x7fffffff || n_channels > 65535)
        return SPK_ERR_ARG;
    if (workspace_bytes < spk_spectrum_stream_finalise_workspace_bytes(n_sel, n_out)) return SPK_ERR_ARG;
    const cudaStream_t st = spk_st(stream);
    double* C = reinterpret_cast<double*>(workspace);
    if (n_sel > 0)
        spk_launch(k_stream_finalise, (unsigned)n_sel, SF_T, 0, st, state, F, n_lags, n, fields, n_out, C);
    spk_launch(k_stream_channels, dim3((unsigned)spk_cdiv(n_out, SC_T), (unsigned)n_channels), SC_T, 0, st,
               (const double*)C, n_out, ch_ptr, weight, acf);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

// Structural observables accumulated inside the captured MD step (DESIGN.md section 24): pair-distance histograms for the
// radial distribution function and mean-squared displacements for self-diffusion.  A one-thread kernel turns the device
// step counter into a flag (step[0] % every == 0) and every later kernel returns at once when it is clear, so one
// captured step serves every step of the run and the cost is paid on sampled steps only.  No float atomics: histograms
// are integer counts and every fp64 sum has a fixed order (segscan.cuh for the per-system sums), so the accumulators are
// bitwise reproducible.
#include <cub/cub.cuh>

#include "cell_grid.cuh"
#include "segscan.cuh"

namespace {

constexpr int RDF_T = 256;          // threads of the histogram traversal (8 warps, one atom per warp at a time)
constexpr int RDF_SMEM_MAX = 48 * 1024;
constexpr int MSD_T = 256;          // atoms per CTA of the MSD partial passes

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// gate[0] = 1 on the steps that sample (step[0] % every == 0, or no step counter), else 0: the one 64-bit modulo of a
// call, so that the kernels after it test a flag
__global__ void k_sample_gate(const int64_t* __restrict__ step, int64_t every, int* __restrict__ gate) {
    SPK_PDL_ENTER();
    gate[0] = step == nullptr || (*step) % every == 0;
}

__device__ __forceinline__ bool gated_off(const int* gate) { return *gate == 0; }

__device__ __forceinline__ double det3(const double* C) {
    return C[0] * (C[4] * C[8] - C[5] * C[7]) - C[1] * (C[3] * C[8] - C[5] * C[6]) + C[2] * (C[3] * C[7] - C[4] * C[6]);
}

// ---- radial distribution function ---------------------------------------------------------------------------------------
// Atoms [a0, a0 + per_cta) per CTA, warp w takes atoms a0 + w, a0 + w + 8, ...; its lanes walk the atoms of the neighbour
// cells exactly as k_nl_search does (same image shifts, same fp32 distance expression), and every pair (i, j, S) with
// |R_j - R_i + S cell| < r_max, (i, j, S) != (i, i, 0), adds 1 to bin floor(d n_bins / r_max) of its species-pair slot
// and of the total slot.  A CTA whose atoms lie in one system counts in a shared-memory histogram [n_slots, n_bins] and
// flushes it with integer atomics; otherwise (or when the histogram does not fit) it counts in global memory directly.
__global__ void __launch_bounds__(RDF_T, 1) k_rdf_traverse(
    const float* __restrict__ R, const int32_t* __restrict__ sys_ptr, int n_sys, int n_atoms,
    const SysGrid* __restrict__ grid, const int* __restrict__ cell_of, const int* __restrict__ wrap,
    const int* __restrict__ sorted_atom, const int* __restrict__ cell_start, const int* __restrict__ cell_end,
    float r_max2, float inv_dr, int n_bins, const int32_t* __restrict__ type, int n_types,
    const int32_t* __restrict__ slot_of, int total_slot, int n_slots, int per_cta, int use_smem,
    unsigned* __restrict__ counts, const int* __restrict__ gate) {
    extern __shared__ unsigned hist[];
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int a0 = blockIdx.x * per_cta;
    if (a0 >= n_atoms) return;
    const int a1 = min(a0 + per_cta, n_atoms);
    const int HB = n_slots * n_bins;
    const int s_first = find_system(sys_ptr, n_sys, a0);
    const bool local = use_smem && find_system(sys_ptr, n_sys, a1 - 1) == s_first;
    if (local)
        for (int k = threadIdx.x; k < HB; k += blockDim.x) hist[k] = 0u;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
    for (int i = a0 + warp; i < a1; i += n_warps) {
        const int s = find_system(sys_ptr, n_sys, i);
        const SysGrid& g = grid[s];
        unsigned* h = local ? hist : counts + (size_t)s * HB;
        const int32_t* row = slot_of + type[i] * n_types;
        const float xi = R[i * 3 + 0], yi = R[i * 3 + 1], zi = R[i * 3 + 2];
        const int wi0 = wrap[i * 3 + 0], wi1 = wrap[i * 3 + 1], wi2 = wrap[i * 3 + 2];
        int lc = cell_of[i] - g.cell_base;
        const int c2 = lc % g.n[2];
        lc /= g.n[2];
        const int c1 = lc % g.n[1], c0 = lc / g.n[1];
        for (int d0 = -g.reach[0]; d0 <= g.reach[0]; ++d0) {
            const int t0 = c0 + d0;
            const int s0 = (t0 >= 0 ? t0 / g.n[0] : -((-t0 + g.n[0] - 1) / g.n[0]));
            const int n0 = t0 - s0 * g.n[0];
            for (int d1 = -g.reach[1]; d1 <= g.reach[1]; ++d1) {
                const int t1 = c1 + d1;
                const int s1 = (t1 >= 0 ? t1 / g.n[1] : -((-t1 + g.n[1] - 1) / g.n[1]));
                const int n1 = t1 - s1 * g.n[1];
                for (int d2 = -g.reach[2]; d2 <= g.reach[2]; ++d2) {
                    const int t2 = c2 + d2;
                    const int s2 = (t2 >= 0 ? t2 / g.n[2] : -((-t2 + g.n[2] - 1) / g.n[2]));
                    const int n2 = t2 - s2 * g.n[2];
                    const int cj = g.cell_base + (n0 * g.n[1] + n1) * g.n[2] + n2;
                    const int end = cell_end[cj];
                    for (int p = cell_start[cj] + lane; p < end; p += 32) {
                        const int j = sorted_atom[p];
                        const int S0 = s0 + wi0 - wrap[j * 3 + 0];
                        const int S1 = s1 + wi1 - wrap[j * 3 + 1];
                        const int S2 = s2 + wi2 - wrap[j * 3 + 2];
                        if (j == i && S0 == 0 && S1 == 0 && S2 == 0) continue;
                        const float ox = (float)S0 * g.c[0] + (float)S1 * g.c[3] + (float)S2 * g.c[6];
                        const float oy = (float)S0 * g.c[1] + (float)S1 * g.c[4] + (float)S2 * g.c[7];
                        const float oz = (float)S0 * g.c[2] + (float)S1 * g.c[5] + (float)S2 * g.c[8];
                        const float dx = R[j * 3 + 0] - xi + ox, dy = R[j * 3 + 1] - yi + oy, dz = R[j * 3 + 2] - zi + oz;
                        const float d2 = dx * dx + dy * dy + dz * dz;
                        if (!(d2 < r_max2)) continue;
                        // d = d2 rsqrt(d2) (a few ulp, no slow-path call of sqrtf); d2 = 0 gives bin 0
                        const int k = min((int)(d2 * rsqrtf(fmaxf(d2, 1e-30f)) * inv_dr), n_bins - 1);
                        const int slot = row[type[j]];
                        if (slot >= 0) atomicAdd(h + slot * n_bins + k, 1u);
                        if (total_slot >= 0) atomicAdd(h + total_slot * n_bins + k, 1u);
                    }
                }
            }
        }
    }
    if (!local) return;
    __syncthreads();
    unsigned* dst = counts + (size_t)s_first * HB;
    for (int k = threadIdx.x; k < HB; k += blockDim.x)
        if (hist[k]) atomicAdd(dst + k, hist[k]);
}

// acc[o, k] += sum_r V_s counts[s, k] over the systems s = r n_out + o (r = 0, 1, ... in order), counts[s, k] = 0;
// volume_sum[o] += sum_r V_s and frames[0] += 1.  V_s = |det(vcell_s)| vscale.
__global__ void __launch_bounds__(256) k_rdf_fold(unsigned* __restrict__ counts, int n_sys, int n_out, int HB,
                                                  const double* __restrict__ vcell, int64_t vstride, double vscale,
                                                  double* __restrict__ acc, double* __restrict__ volume_sum,
                                                  int64_t* __restrict__ frames, const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int o = blockIdx.x;
    const int k = blockIdx.y * blockDim.x + threadIdx.x;
    const int n_rep = n_sys / n_out;
    if (k < HB) {
        double a = acc[(size_t)o * HB + k];
        for (int r = 0; r < n_rep; ++r) {
            const int s = r * n_out + o;
            const double V = fabs(det3(vcell + s * vstride)) * vscale;
            unsigned* c = counts + (size_t)s * HB + k;
            a += V * (double)(*c);
            *c = 0u;
        }
        acc[(size_t)o * HB + k] = a;
    }
    if (blockIdx.y == 0 && threadIdx.x == 0) {
        double v = volume_sum[o];
        for (int r = 0; r < n_rep; ++r) v += fabs(det3(vcell + (r * n_out + o) * vstride)) * vscale;
        volume_sum[o] = v;
        if (o == 0) frames[0] += 1;
    }
}

struct RdfLayout {
    size_t gate, grid, total, cell_of, atom_id, sorted_cell, sorted_atom, wrap, cell_start, cell_end, counts, cub, end;
    size_t cub_bytes;
};

RdfLayout rdf_layout(int64_t n_atoms, int64_t n_sys, int64_t n_slots, int64_t n_bins) {
    RdfLayout L;
    size_t o = 0;
    const size_t ncell = (size_t)(n_atoms + n_sys + 1);
    L.gate = o; o = align256(o + 16);
    L.grid = o; o = align256(o + sizeof(SysGrid) * (size_t)(n_sys > 0 ? n_sys : 1));
    L.total = o; o = align256(o + 16);
    L.cell_of = o; o = align256(o + 4 * (size_t)n_atoms);
    L.atom_id = o; o = align256(o + 4 * (size_t)n_atoms);
    L.sorted_cell = o; o = align256(o + 4 * (size_t)n_atoms);
    L.sorted_atom = o; o = align256(o + 4 * (size_t)n_atoms);
    L.wrap = o; o = align256(o + 12 * (size_t)n_atoms);
    L.cell_start = o; o = align256(o + 4 * ncell);
    L.cell_end = o; o = align256(o + 4 * ncell);
    L.counts = o; o = align256(o + 4 * (size_t)n_sys * (size_t)n_slots * (size_t)n_bins);
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr,
                                    (int)n_atoms);
    L.cub_bytes = sort_b;
    L.cub = o; o = align256(o + L.cub_bytes);
    L.end = o;
    return L;
}

// ---- mean-squared displacement ------------------------------------------------------------------------------------------
// Origin bookkeeping for sample n: origins are taken at samples k origin_every (k = 0, 1, ...) into slot k % n_slots, so
// slot o holds origin k = kmax - ((kmax - o) mod n_slots), kmax = n / origin_every, once kmax >= o.  Returns the lag
// n - k origin_every of slot o, or -1 when the slot is empty or its lag is not kept.
__device__ __forceinline__ int64_t msd_lag(int64_t n, int64_t o, int64_t origin_every, int64_t n_slots, int64_t n_lags) {
    const int64_t kmax = n / origin_every;
    if (kmax < o) return -1;
    const int64_t k = kmax - (kmax - o) % n_slots;
    const int64_t lag = n - k * origin_every;
    return lag < n_lags ? lag : -1;
}

// Per atom: the (centroid) position x in fp64; at the first sample u = last = x, afterwards d = x - last with the
// fractional components of the periodic axes wrapped to [-1/2, 1/2) in the atom's current cell, u += d, last = x.  A
// displacement longer than half the shortest periodic height sets meta[1].  On origin samples u goes to its slot.  CTA 0
// also writes the lag of every origin slot for this sample (lags[o], -1 for none), which the later kernels read.
__global__ void __launch_bounds__(256) k_msd_track(const float* __restrict__ x, int64_t n_atoms, int n_beads,
                                                   const int64_t* __restrict__ idx_m, const double* __restrict__ cell,
                                                   int64_t cell_stride, const uint8_t* __restrict__ pbc,
                                                   int64_t pbc_stride, int64_t origin_every, int64_t n_slots,
                                                   int64_t n_lags, double* __restrict__ track,
                                                   double* __restrict__ origins, int64_t* __restrict__ lags,
                                                   int64_t* __restrict__ meta, const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int64_t n = meta[0];
    if (blockIdx.x == 0)
        for (int64_t o = threadIdx.x; o < n_slots; o += blockDim.x) lags[o] = msd_lag(n, o, origin_every, n_slots, n_lags);
    const int64_t a = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (a >= n_atoms) return;
    double xc[3] = {0.0, 0.0, 0.0};
    for (int r = 0; r < n_beads; ++r)
        for (int j = 0; j < 3; ++j) xc[j] += (double)x[3 * (r * n_atoms + a) + j];
    for (int j = 0; j < 3; ++j) xc[j] /= (double)n_beads;
    double* u = track + 6 * a;
    double* last = u + 3;
    if (n == 0) {
        for (int j = 0; j < 3; ++j) u[j] = last[j] = xc[j];
    } else {
        double d[3] = {xc[0] - last[0], xc[1] - last[1], xc[2] - last[2]};
        const int64_t s = idx_m[a];
        const uint8_t* per = pbc ? pbc + s * pbc_stride : nullptr;
        if (per && (per[0] | per[1] | per[2])) {
            const double* C = cell + s * cell_stride;
            const double det = det3(C);
            const double inv[3][3] = {
                {(C[4] * C[8] - C[5] * C[7]) / det, (C[2] * C[7] - C[1] * C[8]) / det, (C[1] * C[5] - C[2] * C[4]) / det},
                {(C[5] * C[6] - C[3] * C[8]) / det, (C[0] * C[8] - C[2] * C[6]) / det, (C[2] * C[3] - C[0] * C[5]) / det},
                {(C[3] * C[7] - C[4] * C[6]) / det, (C[1] * C[6] - C[0] * C[7]) / det, (C[0] * C[4] - C[1] * C[3]) / det}};
            double shift[3] = {0.0, 0.0, 0.0}, hmin2 = INFINITY;
            for (int j = 0; j < 3; ++j) {
                if (!per[j]) continue;
                const double f = d[0] * inv[0][j] + d[1] * inv[1][j] + d[2] * inv[2][j];
                const double nj = floor(f + 0.5);                   // f - nj in [-1/2, 1/2)
                for (int i = 0; i < 3; ++i) shift[i] += nj * C[j * 3 + i];
                const double il2 = inv[0][j] * inv[0][j] + inv[1][j] * inv[1][j] + inv[2][j] * inv[2][j];
                hmin2 = fmin(hmin2, 1.0 / il2);                      // height_j^2 = 1 / |column j of C^-1|^2
            }
            for (int i = 0; i < 3; ++i) d[i] -= shift[i];
            if (d[0] * d[0] + d[1] * d[1] + d[2] * d[2] > 0.25 * hmin2)
                atomicOr(reinterpret_cast<unsigned long long*>(meta + 1), 1ull);
        }
        for (int j = 0; j < 3; ++j) {
            u[j] += d[j];
            last[j] = xc[j];
        }
    }
    if (n % origin_every == 0) {
        double* uo = origins + ((n / origin_every) % n_slots) * n_atoms * 3 + 3 * a;
        for (int j = 0; j < 3; ++j) uo[j] = u[j];
    }
}

// Per-system sums of m u and m (segmented partial pass of segscan.cuh)
__global__ void __launch_bounds__(MSD_T) k_msd_com_partials(const float* __restrict__ masses,
                                                            const int64_t* __restrict__ idx_m,
                                                            const int32_t* __restrict__ sys_ptr, int64_t n_atoms,
                                                            const double* __restrict__ track,
                                                            double* __restrict__ sys_part, double* __restrict__ head,
                                                            const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int64_t a = (int64_t)blockIdx.x * MSD_T + threadIdx.x;
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    int64_t s = 0, first = 0, end = 0;
    if (a < n_atoms) {
        s = idx_m[a];
        first = sys_ptr[s];
        end = sys_ptr[s + 1];
        const double m = (double)masses[a];
        for (int j = 0; j < 3; ++j) v[j] = m * track[6 * a + j];
        v[3] = m;
    }
    seg_partials<MSD_T, 4>(v, n_atoms, s, first, end, sys_part, head);
}

// com[s] = sum m u / sum m (0 for a massless or empty system); on origin samples also origin_com[slot, s]
__global__ void __launch_bounds__(SEG_FIN_T) k_msd_com_finish(const int32_t* __restrict__ sys_ptr,
                                                              const double* __restrict__ sys_part,
                                                              const double* __restrict__ head, int64_t n_sys,
                                                              int64_t origin_every, int64_t n_slots,
                                                              double* __restrict__ com, double* __restrict__ origin_com,
                                                              const int64_t* __restrict__ meta,
                                                              const int* __restrict__ gate) {
    __shared__ double red[4][SEG_FIN_T];
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int64_t s = blockIdx.x;
    seg_finish_block<MSD_T, 4>(sys_ptr, nullptr, sys_part, head, s, red);
    if (threadIdx.x >= 3) return;
    const int j = threadIdx.x;
    const double m = red[3][0];
    const double c = m > 0.0 ? red[j][0] / m : 0.0;
    com[3 * s + j] = c;
    const int64_t n = meta[0];
    if (n % origin_every == 0) origin_com[((n / origin_every) % n_slots) * n_sys * 3 + 3 * s + j] = c;
}

// CTA (x, o): the squared displacements |u - u_o - (com - com_o)|^2 of its atoms against origin slot o, one column per
// species, into the segmented partials of slot o
template <int NV>
__global__ void __launch_bounds__(MSD_T) k_msd_partials(const int64_t* __restrict__ idx_m,
                                                        const int32_t* __restrict__ sys_ptr,
                                                        const int32_t* __restrict__ species, int64_t n_atoms,
                                                        int64_t n_sys, const double* __restrict__ track,
                                                        const double* __restrict__ origins,
                                                        const double* __restrict__ com,
                                                        const double* __restrict__ origin_com,
                                                        const int64_t* __restrict__ lags,
                                                        double* __restrict__ sys_part, double* __restrict__ head,
                                                        const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int64_t o = blockIdx.y;
    if (lags[o] < 0) return;
    const int64_t a = (int64_t)blockIdx.x * MSD_T + threadIdx.x;
    double v[NV];
#pragma unroll
    for (int c = 0; c < NV; ++c) v[c] = 0.0;
    int64_t s = 0, first = 0, end = 0;
    if (a < n_atoms) {
        s = idx_m[a];
        first = sys_ptr[s];
        end = sys_ptr[s + 1];
        const double* uo = origins + o * n_atoms * 3 + 3 * a;
        double r2 = 0.0;
        for (int j = 0; j < 3; ++j) {
            double d = track[6 * a + j] - uo[j];
            if (com) d -= com[3 * s + j] - origin_com[(o * n_sys + s) * 3 + j];
            r2 += d * d;
        }
        const int sp = species[a];
#pragma unroll
        for (int c = 0; c < NV; ++c) v[c] = c == sp ? r2 : 0.0;
    }
    const int64_t n_cta = gridDim.x;
    seg_partials<MSD_T, NV>(v, n_atoms, s, first, end, sys_part + o * n_sys * NV, head + o * n_cta * NV);
}

// CTA (s, o): acc[s, c, lag(o)] += the sum of system s against slot o, c < n_species
template <int NV>
__global__ void __launch_bounds__(SEG_FIN_T, 1) k_msd_finish(const int32_t* __restrict__ sys_ptr, int64_t n_sys,
                                                          int64_t n_cta, int64_t n_species, int64_t n_lags,
                                                          const int64_t* __restrict__ lags,
                                                          const double* __restrict__ sys_part,
                                                          const double* __restrict__ head, double* __restrict__ acc,
                                                          const int* __restrict__ gate) {
    __shared__ double red[NV][SEG_FIN_T];
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    const int64_t s = blockIdx.x, o = blockIdx.y;
    const int64_t lag = lags[o];
    if (lag < 0) return;
    seg_finish_block<MSD_T, NV>(sys_ptr, nullptr, sys_part + o * n_sys * NV, head + o * n_cta * NV, s, red);
    if (threadIdx.x < n_species) acc[(s * n_species + threadIdx.x) * n_lags + lag] += red[threadIdx.x][0];
}

// count[lag(o)] += 1 for every live slot o, then meta[0] += 1 (the sample is complete)
__global__ void k_msd_advance(int64_t n_slots, const int64_t* __restrict__ lags, int64_t* __restrict__ count,
                              int64_t* __restrict__ meta, const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (gated_off(gate)) return;
    for (int64_t o = threadIdx.x; o < n_slots; o += blockDim.x) {
        const int64_t lag = lags[o];
        if (lag >= 0) count[lag] += 1;
    }
    if (threadIdx.x == 0) meta[0] += 1;
}

int msd_width(int64_t n_species) {
    return n_species <= 1 ? 1 : n_species <= 2 ? 2 : n_species <= 4 ? 4 : 8;
}

struct MsdLayout {
    size_t gate, com_part, com_head, com, lags, part, head, end;
};

MsdLayout msd_layout(int64_t n_atoms, int64_t n_sys, int64_t n_species, int64_t n_slots) {
    MsdLayout L;
    const int64_t n_cta = spk_cdiv(n_atoms, MSD_T), nv = msd_width(n_species);
    size_t o = 0;
    L.gate = o; o += 8;
    L.com_part = o; o += 8 * (size_t)(4 * n_sys);
    L.com_head = o; o += 8 * (size_t)(4 * n_cta);
    L.com = o; o += 8 * (size_t)(3 * n_sys);
    L.lags = o; o += 8 * (size_t)n_slots;
    L.part = o; o += 8 * (size_t)(n_slots * n_sys * nv);
    L.head = o; o += 8 * (size_t)(n_slots * n_cta * nv);
    L.end = o;
    return L;
}

template <int NV>
void msd_launch_sums(dim3 gp, dim3 gf, cudaStream_t st, const int64_t* idx_m, const int32_t* sys_ptr,
                     const int32_t* species, int64_t N, int64_t B, int64_t S, const double* track,
                     const double* origins, const double* com, const double* origin_com, int64_t L,
                     const int64_t* lags, double* part, double* head, double* acc, const int* gate) {
    spk_launch(k_msd_partials<NV>, gp, MSD_T, 0, st, idx_m, sys_ptr, species, N, B, track, origins, com, origin_com, lags,
               part, head, gate);
    spk_launch(k_msd_finish<NV>, gf, SEG_FIN_T, 0, st, sys_ptr, B, (int64_t)gp.x, S, L, lags, (const double*)part,
               (const double*)head, acc, gate);
}

}  // namespace

extern "C" size_t spk_rdf_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n_slots, int64_t n_bins) {
    if (n_atoms < 0 || n_sys < 0 || n_slots < 0 || n_bins < 0) return 0;
    return rdf_layout(n_atoms, n_sys, n_slots, n_bins).end;
}

extern "C" int spk_rdf_accumulate(const float* R, const float* cell, const uint8_t* pbc, const int32_t* sys_ptr,
                                  int64_t n_atoms, int64_t n_sys, const int32_t* type, int64_t n_types,
                                  const int32_t* slot_of, int32_t total_slot, int64_t n_slots, float r_max,
                                  int64_t n_bins, const double* volume_cell, int64_t volume_cell_stride,
                                  double volume_scale, int64_t n_out, const int64_t* step, int64_t every, double* acc,
                                  double* volume_sum, int64_t* frames, void* workspace, size_t workspace_bytes,
                                  spk_stream_t stream) {
    if (n_atoms < 0 || n_sys < 1 || n_types < 1 || n_slots < 1 || n_bins < 1 || !(r_max > 0.f) || every < 1) return SPK_ERR_ARG;
    if (n_out < 1 || n_sys % n_out != 0 || total_slot < -1 || total_slot >= n_slots) return SPK_ERR_ARG;
    if (volume_cell_stride != 0 && volume_cell_stride != 9) return SPK_ERR_ARG;
    if (n_atoms > 0x3fffffff || n_slots * n_bins > 0x3fffffff || n_sys * n_slots * n_bins > 0x3fffffff)
        return SPK_ERR_UNSUPPORTED;
    if (!R || !cell || !pbc || !sys_ptr || !type || !slot_of || !volume_cell || !acc || !volume_sum || !frames || !workspace)
        return SPK_ERR_ARG;
    const RdfLayout L = rdf_layout(n_atoms, n_sys, n_slots, n_bins);
    if (workspace_bytes < L.end) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    int* gate = reinterpret_cast<int*>(ws + L.gate);
    SysGrid* grid = reinterpret_cast<SysGrid*>(ws + L.grid);
    int* total = reinterpret_cast<int*>(ws + L.total);
    int* cell_of = reinterpret_cast<int*>(ws + L.cell_of);
    int* atom_id = reinterpret_cast<int*>(ws + L.atom_id);
    int* sorted_cell = reinterpret_cast<int*>(ws + L.sorted_cell);
    int* sorted_atom = reinterpret_cast<int*>(ws + L.sorted_atom);
    int* wrap = reinterpret_cast<int*>(ws + L.wrap);
    int* cell_start = reinterpret_cast<int*>(ws + L.cell_start);
    int* cell_end = reinterpret_cast<int*>(ws + L.cell_end);
    unsigned* counts = reinterpret_cast<unsigned*>(ws + L.counts);
    const int N = (int)n_atoms, B = (int)n_sys, HB = (int)(n_slots * n_bins);
    spk_launch(k_sample_gate, 1, 1, 0, st, step, every, gate);
    if (N > 0) {
        cudaError_t e = cudaMemsetAsync(ws + L.cell_start, 0, L.counts - L.cell_start, st);   // empty cells: start == end
        if (e != cudaSuccess) return SPK_CUDA_ERR(e);
        spk_launch(k_nl_setup, 1, 1024, 0, st, cell, pbc, sys_ptr, B, r_max, grid, total, gate);
        spk_launch(k_nl_bin, (unsigned)spk_cdiv(N, 256), 256, 0, st, R, sys_ptr, B, N, (const SysGrid*)grid, cell_of,
                   atom_id, wrap, gate);
        size_t cub_bytes = L.cub_bytes;
        e = cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, (const int*)cell_of, sorted_cell, (const int*)atom_id,
                                            sorted_atom, N, 0, 32, st);
        if (e != cudaSuccess) return SPK_CUDA_ERR(e);
        spk_launch(k_nl_cell_bounds, (unsigned)spk_cdiv(N, 256), 256, 0, st, (const int*)sorted_cell, N, cell_start,
                   cell_end, gate);
        const int per_cta = (int)std::max<int64_t>(16, spk_cdiv(N, 4 * SPK_NUM_SMS));
        const size_t smem = (size_t)HB * 4;
        const int use_smem = smem <= (size_t)RDF_SMEM_MAX ? 1 : 0;
        const float dr = r_max / (float)n_bins;
        spk_launch(k_rdf_traverse, (unsigned)spk_cdiv(N, per_cta), RDF_T, use_smem ? smem : 0, st, R, sys_ptr, B, N,
                   (const SysGrid*)grid, (const int*)cell_of, (const int*)wrap, (const int*)sorted_atom,
                   (const int*)cell_start, (const int*)cell_end, r_max * r_max, 1.0f / dr, (int)n_bins, type,
                   (int)n_types, slot_of, (int)total_slot, (int)n_slots, per_cta, use_smem, counts, gate);
    }
    spk_launch(k_rdf_fold, dim3((unsigned)n_out, (unsigned)spk_cdiv(HB, 256)), 256, 0, st, counts, B, (int)n_out, HB,
               volume_cell, volume_cell_stride, volume_scale, acc, volume_sum, frames, gate);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" size_t spk_msd_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n_species, int64_t n_slots) {
    if (n_atoms < 0 || n_sys < 0 || n_species < 1 || n_species > 8 || n_slots < 1) return 0;
    return msd_layout(n_atoms, n_sys, n_species, n_slots).end;
}

extern "C" int spk_msd_accumulate(const float* positions, int64_t n_atoms, int32_t n_beads, const float* masses,
                                  const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_sys, const int32_t* species,
                                  int64_t n_species, const double* cell, int64_t cell_stride, const uint8_t* pbc,
                                  int64_t pbc_stride, int remove_com, int64_t n_lags, int64_t origin_every,
                                  int64_t n_slots, const int64_t* step, int64_t every, double* track, double* origins,
                                  double* origin_com, double* acc, int64_t* count, int64_t* meta, void* workspace,
                                  size_t workspace_bytes, spk_stream_t stream) {
    if (n_atoms < 1 || n_beads < 1 || n_sys < 1 || n_lags < 1 || origin_every < 1 || every < 1) return SPK_ERR_ARG;
    if (n_species < 1 || n_slots != spk_cdiv(n_lags, origin_every)) return SPK_ERR_ARG;
    if (n_species > 8) return SPK_ERR_UNSUPPORTED;
    if (n_atoms * n_beads >= (1ll << 31) / 3) return SPK_ERR_UNSUPPORTED;
    if ((cell_stride != 0 && cell_stride != 9) || (pbc_stride != 0 && pbc_stride != 3) || (pbc && !cell)) return SPK_ERR_ARG;
    if (!positions || !idx_m || !sys_ptr || !species || !track || !origins || !acc || !count || !meta || !workspace)
        return SPK_ERR_ARG;
    if (remove_com && (!masses || !origin_com)) return SPK_ERR_ARG;
    const MsdLayout L = msd_layout(n_atoms, n_sys, n_species, n_slots);
    if (workspace_bytes < L.end) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    int* gate = reinterpret_cast<int*>(ws + L.gate);
    double* com_part = reinterpret_cast<double*>(ws + L.com_part);
    double* com_head = reinterpret_cast<double*>(ws + L.com_head);
    double* com = remove_com ? reinterpret_cast<double*>(ws + L.com) : nullptr;
    int64_t* lags = reinterpret_cast<int64_t*>(ws + L.lags);
    double* part = reinterpret_cast<double*>(ws + L.part);
    double* head = reinterpret_cast<double*>(ws + L.head);
    const int64_t n_cta = spk_cdiv(n_atoms, MSD_T);
    spk_launch(k_sample_gate, 1, 1, 0, st, step, every, gate);
    spk_launch(k_msd_track, (unsigned)spk_cdiv(n_atoms, 256), 256, 0, st, positions, n_atoms, (int)n_beads, idx_m, cell,
               cell_stride, pbc, pbc_stride, origin_every, n_slots, n_lags, track, origins, lags, meta, gate);
    if (remove_com) {
        spk_launch(k_msd_com_partials, (unsigned)n_cta, MSD_T, 0, st, masses, idx_m, sys_ptr, n_atoms,
                   (const double*)track, com_part, com_head, gate);
        spk_launch(k_msd_com_finish, (unsigned)n_sys, SEG_FIN_T, 0, st, sys_ptr, (const double*)com_part,
                   (const double*)com_head, n_sys, origin_every, n_slots, com, origin_com, (const int64_t*)meta, gate);
    }
    const dim3 gp((unsigned)n_cta, (unsigned)n_slots), gf((unsigned)n_sys, (unsigned)n_slots);
    const int nv = msd_width(n_species);
    const double* oc = remove_com ? origin_com : nullptr;
    if (nv == 1)
        msd_launch_sums<1>(gp, gf, st, idx_m, sys_ptr, species, n_atoms, n_sys, n_species, track, origins, com, oc,
                           n_lags, lags, part, head, acc, gate);
    else if (nv == 2)
        msd_launch_sums<2>(gp, gf, st, idx_m, sys_ptr, species, n_atoms, n_sys, n_species, track, origins, com, oc,
                           n_lags, lags, part, head, acc, gate);
    else if (nv == 4)
        msd_launch_sums<4>(gp, gf, st, idx_m, sys_ptr, species, n_atoms, n_sys, n_species, track, origins, com, oc,
                           n_lags, lags, part, head, acc, gate);
    else
        msd_launch_sums<8>(gp, gf, st, idx_m, sys_ptr, species, n_atoms, n_sys, n_species, track, origins, com, oc,
                           n_lags, lags, part, head, acc, gate);
    spk_launch(k_msd_advance, 1, 256, 0, st, n_slots, (const int64_t*)lags, count, meta, gate);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

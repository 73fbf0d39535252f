// SchNet continuous-filter convolution kernels and Atomwise head.
// Reference: representation/schnet.py:62-67 (Wij * rcut, x[idx_j], x_j * Wij, scatter_add), atomistic/atomwise.py:69-88.
// Thread c of a CTA owns feature channel c; CTAs take edge-balanced contiguous row ranges; reductions over a
// receiver's (or sender's) edges are private register accumulations -> deterministic, no atomics.
#include "common.cuh"

namespace {

constexpr int CH = 32;

template <int NW>
__global__ void __launch_bounds__(NW * 32) k_cfconv_fwd(const float* __restrict__ h, const float* __restrict__ w_raw,
                                                        const float* __restrict__ geo, const int* __restrict__ rowptr,
                                                        const int* __restrict__ slot_j, int n_atoms, int n_edges,
                                                        float* __restrict__ m) {
    SPK_PDL_ENTER();
    constexpr int F = NW * 32;
    const int c = threadIdx.x;
    const int row_lo = spk_block_row_begin(rowptr, n_atoms, n_edges, gridDim.x, blockIdx.x);
    const int row_hi = spk_block_row_begin(rowptr, n_atoms, n_edges, gridDim.x, blockIdx.x + 1);
    for (int i = row_lo; i < row_hi; ++i) {
        float acc = 0.f;
        const int s0 = rowptr[i], s1 = rowptr[i + 1];
#pragma unroll 4
        for (int s = s0; s < s1; ++s) {
            const int j = slot_j[s];
            const float fc = geo[(int64_t)s * SPK_GEO_STRIDE + 4];
            acc = fmaf(h[(int64_t)j * F + c], w_raw[(int64_t)s * F + c] * fc, acc);
        }
        m[(int64_t)i * F + c] = acc;
    }
}

template <int NW>
__global__ void __launch_bounds__(NW * 32) k_cfconv_bwd(const float* __restrict__ h, const float* __restrict__ w_raw,
                                                        const float* __restrict__ geo, const float* __restrict__ g_m,
                                                        const int* __restrict__ sptr, const int* __restrict__ pos_slot,
                                                        const int* __restrict__ pos_i, int n_atoms, int n_edges,
                                                        float* __restrict__ g_h, float* __restrict__ g_wraw,
                                                        float* __restrict__ g_fc) {
    SPK_PDL_ENTER();
    constexpr int F = NW * 32;
    __shared__ float s_red[CH][NW];
    __shared__ int s_slot[CH];
    const int c = threadIdx.x, lane = c & 31, warp = c >> 5;
    const int j_lo = spk_block_row_begin(sptr, n_atoms, n_edges, gridDim.x, blockIdx.x);
    const int j_hi = spk_block_row_begin(sptr, n_atoms, n_edges, gridDim.x, blockIdx.x + 1);
    if (j_lo >= j_hi) return;
    const int p_begin = sptr[j_lo], p_end = sptr[j_hi];
    int j = j_lo;
    int next_boundary = sptr[j + 1];
    float hj = h[(int64_t)j * F + c];
    float acc = 0.f;
    for (int cs = p_begin; cs < p_end; cs += CH) {
        const int n = min(CH, p_end - cs);
        __syncthreads();
        for (int t = 0; t < n; ++t) {
            const int p = cs + t;
            if (p >= next_boundary) {
                do {
                    g_h[(int64_t)j * F + c] = acc;
                    acc = 0.f;
                    ++j;
                    next_boundary = sptr[j + 1];
                } while (p >= next_boundary);
                hj = h[(int64_t)j * F + c];
            }
            const int s = pos_slot[p];
            const int i = pos_i[p];
            const float fc = geo[(int64_t)s * SPK_GEO_STRIDE + 4];
            const float gm = g_m[(int64_t)i * F + c];
            const float wr = w_raw[(int64_t)s * F + c];
            acc = fmaf(wr * fc, gm, acc);
            const float hg = hj * gm;
            g_wraw[(int64_t)s * F + c] = hg * fc;
            float part = spk_warp_sum(hg * wr);
            if (lane == 0) s_red[t][warp] = part;
            if (c == 0) s_slot[t] = s;
        }
        __syncthreads();
        if (threadIdx.x < n) {
            float v = 0.f;
#pragma unroll
            for (int wv = 0; wv < NW; ++wv) v += s_red[threadIdx.x][wv];
            g_fc[s_slot[threadIdx.x]] = v;
        }
    }
    for (; j < j_hi; ++j) {
        g_h[(int64_t)j * F + c] = acc;
        acc = 0.f;
    }
}

__global__ void k_radial_bwd(const float* __restrict__ g_phi, const float* __restrict__ g_fc,
                             const float* __restrict__ dphi, const float* __restrict__ geo,
                             const int* __restrict__ slot_eid, int64_t n_edges, int n_rbf, int KP,
                             float* __restrict__ g_rij, int accumulate) {
    SPK_PDL_ENTER();
    int64_t s = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (s >= n_edges) return;
    float gd = 0.f;
    if (g_phi)
        for (int k = 0; k < n_rbf; ++k) gd = fmaf(g_phi[s * KP + k], dphi[s * KP + k], gd);
    const float* ge = geo + s * SPK_GEO_STRIDE;
    if (g_fc) gd = fmaf(g_fc[s], ge[5], gd);
    int64_t e = slot_eid ? (int64_t)slot_eid[s] : s;
    float r0 = gd * ge[0], r1 = gd * ge[1], r2 = gd * ge[2];
    if (accumulate) {
        r0 += g_rij[e * 3 + 0];
        r1 += g_rij[e * 3 + 1];
        r2 += g_rij[e * 3 + 2];
    }
    g_rij[e * 3 + 0] = r0;
    g_rij[e * 3 + 1] = r1;
    g_rij[e * 3 + 2] = r2;
}

// y[a] = hid[a,:] . w1 + b1 : one warp per atom
__global__ void k_atom_dot(const float* __restrict__ hid, const float* __restrict__ w1, const float* __restrict__ b1,
                           int64_t n_atoms, int H, float* __restrict__ y) {
    SPK_PDL_ENTER();
    int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (warp >= n_atoms) return;
    float acc = 0.f;
    for (int k = lane; k < H; k += 32) acc = fmaf(hid[warp * H + k], w1[k], acc);
    acc = spk_warp_sum(acc);
    if (lane == 0) y[warp] = acc + (b1 ? b1[0] : 0.f);
}

// energy[m] = sum_{a in [mol_ptr[m], mol_ptr[m+1])} y[a] : one 256-thread CTA per system, fixed reduction tree
__global__ void __launch_bounds__(256) k_mol_sum(const float* __restrict__ y, const int* __restrict__ mol_ptr,
                                                 float* __restrict__ energy) {
    SPK_PDL_ENTER();
    __shared__ float s_w[8];
    const int m = blockIdx.x;
    const int a0 = mol_ptr[m], a1 = mol_ptr[m + 1];
    float acc = 0.f;
    for (int a = a0 + threadIdx.x; a < a1; a += 256) acc += y[a];
    acc = spk_warp_sum(acc);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float v = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) v += s_w[k];
        energy[m] = v;
    }
}

__global__ void k_atomwise_out_bwd(const float* __restrict__ g_energy, const int64_t* __restrict__ idx_m,
                                   const float* __restrict__ w1, int64_t n_atoms, int H, float* __restrict__ g_hid) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * H) return;
    int64_t a = t / H;
    int k = (int)(t - a * H);
    float g = g_energy ? g_energy[idx_m[a]] : 1.0f;
    g_hid[t] = g * w1[k];
}

}  // namespace

#define GRID1D(n, T) (unsigned)spk_cdiv((n), (T)), (T), 0, spk_st(stream)

extern "C" int spk_cfconv_fwd(const float* h, const float* w_raw, const float* geo, const int32_t* rowptr,
                              const int32_t* slot_j, int64_t n_atoms, int64_t n_edges, int F, float* m,
                              spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0) return SPK_ERR_ARG;
    if ((F & 31) || F > 256) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!h || !rowptr || !m) return SPK_ERR_ARG;
    if (n_edges > 0 && (!w_raw || !geo || !slot_j)) return SPK_ERR_ARG;
    int64_t nb = spk_cdiv(n_edges, 128);
    if (nb < 1) nb = 1;
    if (nb > n_atoms) nb = n_atoms;
    cudaStream_t st = spk_st(stream);
    int na = (int)n_atoms, ne = (int)n_edges;
    switch (F / 32) {
        case 1: spk_launch(k_cfconv_fwd<1>, (unsigned)nb, 32, 0, st, h, w_raw, geo, rowptr, slot_j, na, ne, m); break;
        case 2: spk_launch(k_cfconv_fwd<2>, (unsigned)nb, 64, 0, st, h, w_raw, geo, rowptr, slot_j, na, ne, m); break;
        case 4: spk_launch(k_cfconv_fwd<4>, (unsigned)nb, 128, 0, st, h, w_raw, geo, rowptr, slot_j, na, ne, m); break;
        case 8: spk_launch(k_cfconv_fwd<8>, (unsigned)nb, 256, 0, st, h, w_raw, geo, rowptr, slot_j, na, ne, m); break;
        default: return SPK_ERR_UNSUPPORTED;
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_cfconv_bwd(const float* h, const float* w_raw, const float* geo, const float* g_m,
                              const int32_t* sptr, const int32_t* pos_slot, const int32_t* pos_i, int64_t n_atoms,
                              int64_t n_edges, int F, float* g_h, float* g_wraw, float* g_fc, spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0) return SPK_ERR_ARG;
    if ((F & 31) || F > 256) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!h || !g_m || !sptr || !g_h) return SPK_ERR_ARG;
    if (n_edges > 0 && (!w_raw || !geo || !pos_slot || !pos_i || !g_wraw || !g_fc)) return SPK_ERR_ARG;
    int64_t nb = spk_cdiv(n_edges, 128);
    if (nb < 1) nb = 1;
    if (nb > n_atoms) nb = n_atoms;
    cudaStream_t st = spk_st(stream);
    int na = (int)n_atoms, ne = (int)n_edges;
    switch (F / 32) {
        case 1: spk_launch(k_cfconv_bwd<1>, (unsigned)nb, 32, 0, st, h, w_raw, geo, g_m, sptr, pos_slot, pos_i, na, ne, g_h, g_wraw, g_fc); break;
        case 2: spk_launch(k_cfconv_bwd<2>, (unsigned)nb, 64, 0, st, h, w_raw, geo, g_m, sptr, pos_slot, pos_i, na, ne, g_h, g_wraw, g_fc); break;
        case 4: spk_launch(k_cfconv_bwd<4>, (unsigned)nb, 128, 0, st, h, w_raw, geo, g_m, sptr, pos_slot, pos_i, na, ne, g_h, g_wraw, g_fc); break;
        case 8: spk_launch(k_cfconv_bwd<8>, (unsigned)nb, 256, 0, st, h, w_raw, geo, g_m, sptr, pos_slot, pos_i, na, ne, g_h, g_wraw, g_fc); break;
        default: return SPK_ERR_UNSUPPORTED;
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_radial_bwd(const float* g_phi, const float* g_fc, const float* dphi, const float* geo,
                              const int32_t* slot_eid, int64_t n_edges, int n_rbf, float* g_rij, int accumulate,
                              spk_stream_t stream) {
    if (n_edges < 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (n_rbf > 32) return SPK_ERR_UNSUPPORTED;
    if (n_edges == 0) return SPK_OK;
    if (!geo || !g_rij || (g_phi && !dphi)) return SPK_ERR_ARG;
    spk_launch(k_radial_bwd, GRID1D(n_edges, 256), g_phi, g_fc, dphi, geo, slot_eid, n_edges, n_rbf, spk_kp(n_rbf), g_rij,
                                           accumulate);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_atomwise_out(const float* hid, const float* w1, const float* b1, const int32_t* mol_ptr,
                                int64_t n_atoms, int64_t n_mol, int H, float* y, float* energy, spk_stream_t stream) {
    if (n_atoms < 0 || n_mol < 0 || H <= 0) return SPK_ERR_ARG;
    if (n_atoms > 0) {
        if (!hid || !w1 || !y) return SPK_ERR_ARG;
        spk_launch(k_atom_dot, GRID1D(n_atoms * 32, 256), hid, w1, b1, n_atoms, H, y);
    }
    if (energy && n_mol > 0) {
        if (!mol_ptr) return SPK_ERR_ARG;
        spk_launch(k_mol_sum, (unsigned)n_mol, 256, 0, spk_st(stream), y, mol_ptr, energy);
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_atomwise_out_bwd(const float* g_energy, const int64_t* idx_m, const float* w1, int64_t n_atoms,
                                    int H, float* g_hid, spk_stream_t stream) {
    if (n_atoms < 0 || H <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!w1 || !g_hid || (g_energy && !idx_m)) return SPK_ERR_ARG;
    spk_launch(k_atomwise_out_bwd, GRID1D(n_atoms * H, 256), g_energy, idx_m, w1, n_atoms, H, g_hid);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

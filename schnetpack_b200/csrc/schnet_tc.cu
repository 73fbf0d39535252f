// SchNet interaction block, forward, as ONE fused edge kernel with the filter network on the tensor cores (wgmma).
// Reference: representation/schnet.py
//     Wij = filter_network(f_ij) * rcut_ij        filter_network = Dense(n_rbf -> F, ssp) -> Dense(F -> F)
//     x   = scatter_add( x[idx_j] * Wij, idx_i )
// The reference materialises the [E,F] hidden layer and the [E,F] filter in HBM per block (2 x 512 B per edge and layer,
// round trips included ~2 KB) -- 38 kFLOP per edge and layer of dense work.  Here a chunk of 32 edges goes through both
// layers without leaving the SM:
//
//   producers   Phi' = [phi | 1 | 0] rows of the chunk (hi/lo TF32 split) -> shared memory (K-major, 64 B swizzle);
//   groups      4 consumer warpgroups; group g owns 8 edges of every chunk (and its own edge-balanced receiver range).  It
//               computes with wgmma, 3xTF32 (small products first; wgmma.cuh):
//       MMA 1   H = [W0 | b0] Phi'_g^T       128 hidden channels (two m64 halves) x 8 edges, K = n_rbf + 1;
//       act     shifted softplus on the fragment registers, hi/lo split, written as the group's 8 rows of the K-major
//               B operand of the second layer (only this warpgroup reads them);
//       MMA 2   D = W1 ssp(H)                 128 output channels x 8 edges, K = 128: the main products in one accumulator,
//               the small hi*lo terms in a second one (the tensor core truncates when it accumulates);
//       gather  D goes through a small shared-memory transpose to thread = channel; filter value
//               W = (D + b1) * fc, gather h[j, c], accumulate the receiver's row in registers (CSR order, deterministic, no
//               atomics), m[i] on flush.
//
// Both weight operands ([W0|b0]: 32 KB, W1: 128 KB as hi|lo tiles) stay resident in shared memory for the life of the
// persistent CTA (one per SM) and arrive by two TMA bulk copies.  The receiver ranges come from a CSR that may have been
// built from the ACTIVE edges only (spk_graph_build_active: d < cutoff), so the padding slots of a padded neighbour list
// cost nothing -- their filter is exactly 0 in the reference (nn/cutoff.py).
// The reverse pass (forces) keeps the materialised-filter pipeline: the named SchNet workload with forces is the 9-atom cfg1;
// cfg3 is energy-only inference.
#include "wgmma.cuh"

namespace {

constexpr int F_TC = 128;
constexpr int EG = 8, NG = 4, NE = EG * NG;              // 32 edge rows per chunk, 8 per group (wgmma N)
constexpr int NCW = NG * 4;                              // 16 consumer warps = 4 warpgroups
constexpr int W_PROD0 = NCW;
constexpr int NPROD = 2, NST = 2;                        // Phi' stages (chunk k -> stage k % 2 -> producer k % 2)
constexpr int NMETA = 4;                                 // (sender, fc) ring
constexpr int NTHREADS = (W_PROD0 + NPROD) * 32;         // 576
constexpr int KT = 16;
constexpr int A_TILE = F_TC * KT * 4;                    // 8192 B
constexpr int W0_BYTES = 2 * 2 * A_TILE;                 // [hi,lo][2 k-tiles]
constexpr int W1_BYTES = 2 * 8 * A_TILE;                 // [hi,lo][8 k-tiles]
constexpr int B_TILE = NE * KT * 4;                      // 2048 B
constexpr int PHI_STAGE = 2 * 2 * B_TILE;                // [hi,lo][2 k-tiles]
constexpr int B2_BYTES = 2 * 8 * B_TILE;                 // [hi,lo][8 k-tiles]
constexpr int META_STAGE = NE * 8;                       // int sender + float fc per row
constexpr int T_LD = F_TC + 4;                           // row of the per-group transpose tile [edge][channel] (floats)
constexpr int T_BYTES = NG * EG * T_LD * 4;
// the 64-byte swizzle repeats every 512 B, so 512 B alignment suffices; the static shared variables round up to the same
// 512 B and count against the 227 KB a block may use
constexpr int SMEM_ALIGN = 512;
constexpr int SMEM_BYTES = W0_BYTES + W1_BYTES + NST * PHI_STAGE + B2_BYTES + NMETA * META_STAGE + T_BYTES + SMEM_ALIGN;
static_assert(SMEM_BYTES + SMEM_ALIGN <= 227 * 1024, "shared memory budget (dynamic + static)");

// packed operands: [W0|b0|0] as [hi,lo][2 k-tiles][128 x 16], then W1 as [hi,lo][8 k-tiles][128 x 16]
__global__ void k_pack_schnet_filter(const float* __restrict__ w0, const float* __restrict__ b0,
                                     const float* __restrict__ w1, int n_rbf, float* __restrict__ out) {
    SPK_PDL_WAIT_ONLY();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    constexpr int N0 = F_TC * 32, N1 = F_TC * F_TC;
    if (t >= N0 + N1) return;
    float w;
    int row, k, nkt;
    float* base;
    if (t < N0) {
        k = t & 31;
        row = t >> 5;
        w = k < n_rbf ? w0[(int64_t)row * n_rbf + k] : (k == n_rbf ? b0[row] : 0.f);
        nkt = 2;
        base = out;
    } else {
        const int u = t - N0;
        k = u & (F_TC - 1);
        row = u >> 7;
        w = w1[(int64_t)row * F_TC + k];
        nkt = 8;
        base = out + W0_BYTES / 4;
    }
    const float hi = tf32_rn(w), lo = w - hi;
    const int kt = k >> 4, kk = k & 15;
    const int off = tile_off(row, kk >> 2) / 4 + (kk & 3);
    base[(0 * nkt + kt) * (A_TILE / 4) + off] = hi;
    base[(1 * nkt + kt) * (A_TILE / 4) + off] = lo;
}

__global__ void __launch_bounds__(NTHREADS, 1) k_schnet_cfconv_fwd_tc(
    const float* __restrict__ h, const float* __restrict__ phi, const float* __restrict__ geo,
    const int* __restrict__ rowptr, const int* __restrict__ slot_j, const float* __restrict__ wpk,
    const float* __restrict__ b1, int act, int n_atoms, int n_rbf, float* __restrict__ m) {
    constexpr int F = F_TC;
    extern __shared__ __align__(SMEM_ALIGN) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((SMEM_ALIGN - (smem_u32(smem_raw) & (SMEM_ALIGN - 1))) & (SMEM_ALIGN - 1));
    uint8_t* sW0 = smem;
    uint8_t* sW1 = sW0 + W0_BYTES;
    uint8_t* sPhi = sW1 + W1_BYTES;
    uint8_t* sB2 = sPhi + NST * PHI_STAGE;
    uint8_t* sMeta = sB2 + B2_BYTES;
    float* sT = reinterpret_cast<float*>(sMeta + NMETA * META_STAGE);
    __shared__ __align__(8) uint64_t w_full, phi_full[NST], phi_empty[NST], meta_full[NMETA], meta_empty[NMETA];
    __shared__ int s_rlo[NG], s_rhi[NG], s_sb[NG], s_se[NG];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) {
        mbar_init(&w_full, 1);
#pragma unroll
        for (int s = 0; s < NST; ++s) {
            mbar_init(&phi_full[s], 1);
            mbar_init(&phi_empty[s], NCW);
        }
#pragma unroll
        for (int s = 0; s < NMETA; ++s) {
            mbar_init(&meta_full[s], 1);
            mbar_init(&meta_empty[s], NCW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&w_full, W0_BYTES + W1_BYTES);      // static operand: fetched BEFORE griddepcontrol.wait (pack kernels never trigger their dependents early, common.cuh)
        tma_load(sW0, wpk, W0_BYTES, &w_full);
        tma_load(sW1, wpk + W0_BYTES / 4, W1_BYTES, &w_full);
    }
    SPK_PDL_WAIT();
    if (warp <= NG) {                              // warp w finds boundary w of this CTA's NG group ranges (warp-wide search)
        const int n_act = rowptr[n_atoms];                  // edges in the (possibly active-only) CSR
        const int bnd = spk_block_row_begin_warp(rowptr, n_atoms, n_act, gridDim.x * NG, blockIdx.x * NG + warp);
        if (lane == 0) {
            const int e = rowptr[bnd];
            if (warp < NG) {
                s_rlo[warp] = bnd;
                s_sb[warp] = e;
            }
            if (warp > 0) {
                s_rhi[warp - 1] = bnd;
                s_se[warp - 1] = e;
            }
        }
    }
    __syncthreads();
    int n_chunks = 0;
#pragma unroll
    for (int g = 0; g < NG; ++g) n_chunks = max(n_chunks, (s_se[g] - s_sb[g] + EG - 1) / EG);
    const int KP = spk_kp(n_rbf);
    const int nks1 = (n_rbf + 1 + 7) >> 3;                  // k-steps of the first layer (K = n_rbf + 1 padded to 8)

    if (warp >= W_PROD0) {
        // =========================================== producers ===========================================
        const int p = warp - W_PROD0;
        const int qc = lane & 7, rsub = lane >> 3;          // 8 x 16 B chunks per row (32 floats), 4 rows per pass, 8 passes
        const bool q_in = qc * 4 < KP;
        const int kb_chunk = n_rbf >> 2, kb = n_rbf & 3;    // the bias column k = n_rbf
        for (int k = p; k < n_chunks; k += NPROD) {
            const int st = k % NST, use = k / NST;
            const int ms = k % NMETA, muse = k / NMETA;
            uint8_t* stP = sPhi + st * PHI_STAGE;
            int* st_j = reinterpret_cast<int*>(sMeta + ms * META_STAGE);
            float* st_fc = reinterpret_cast<float*>(sMeta + ms * META_STAGE + NE * 4);
            // unconditional clamped loads, issued before the waits (rows past a group's end read slot 0, zeroed below)
            const int g0 = lane / EG;
            const int s0 = s_sb[g0] + k * EG + (lane % EG);
            const bool ok0 = s0 < s_se[g0];
            const int sl0 = ok0 ? s0 : 0;
            const int mj = slot_j[sl0];
            const float mfc = geo[(int64_t)sl0 * SPK_GEO_STRIDE + 4];
            float4 pv[8];
            bool okv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = i * 4 + rsub, g = r / EG;
                const int s = s_sb[g] + k * EG + (r % EG);
                okv[i] = s < s_se[g];
                const int sl = okv[i] ? s : 0;
                pv[i] = *reinterpret_cast<const float4*>(phi + (int64_t)sl * KP + (q_in ? qc * 4 : 0));
            }
            if (use >= 1) mbar_wait(&phi_empty[st], (use - 1) & 1);
            if (muse >= 1) mbar_wait(&meta_empty[ms], (muse - 1) & 1);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int r = i * 4 + rsub;
                float4 v = q_in ? pv[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                if (qc == kb_chunk) {
                    if (kb == 0) v.x = 1.f; else if (kb == 1) v.y = 1.f; else if (kb == 2) v.z = 1.f; else v.w = 1.f;
                }
                if (!okv[i]) v = make_float4(0.f, 0.f, 0.f, 0.f);
                float4 hi, lo;
                hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
                lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
                const int off = tile_off(r, qc & 3);
                *reinterpret_cast<float4*>(stP + ((qc >> 2) * 2 + 0) * B_TILE + off) = hi;     // [k-tile][hi | lo]
                *reinterpret_cast<float4*>(stP + ((qc >> 2) * 2 + 1) * B_TILE + off) = lo;
            }
            st_j[lane] = mj;
            st_fc[lane] = ok0 ? mfc : 0.f;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) {
                mbar_arrive(&phi_full[st]);
                mbar_arrive(&meta_full[ms]);
            }
        }
    } else {
        // =========================================== consumer warpgroups ===========================================
        const int g = warp >> 2;
        const int c = tid & 127;                                       // channel of the gather / accumulate phase
        const float b1c = b1 ? b1[c] : 0.f;
        const int row_hi = s_rhi[g], s_begin = s_sb[g], s_end = s_se[g];
        int i = s_rlo[g];
        int next_boundary = i < row_hi ? rowptr[i + 1] : 0x7fffffff;
        float acc = 0.f;
        float* tg = sT + g * EG * T_LD;                                // this group's [edge][channel] transpose tile
        const uint32_t a0 = smem_u32(sW0), a1 = smem_u32(sW1), bb2 = smem_u32(sB2) + (uint32_t)(g * EG * SPK_SW64_ROW);
        mbar_wait(&w_full, 0);
        for (int k = 0; k < n_chunks; ++k) {
            const int st = k % NST, ms = k % NMETA;
            // ---- MMA 1: H = [W0|b0] Phi'^T for the group's 8 edges
            mbar_wait(&phi_full[st], (k / NST) & 1);
            const uint32_t bp = smem_u32(sPhi + st * PHI_STAGE) + (uint32_t)(g * EG * SPK_SW64_ROW);
            float hf[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            wgmma_fence();
            for (int s3 = 0; s3 < nks1; ++s3) {
                const int kt = s3 >> 1, ko = (s3 & 1) * 32;
#pragma unroll
                for (int mh = 0; mh < 2; ++mh) {
                    const uint32_t ah = a0 + (0 * 2 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko;
                    const uint32_t al = a0 + (1 * 2 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko;
                    const uint32_t bh = bp + (kt * 2 + 0) * B_TILE + ko, bl = bp + (kt * 2 + 1) * B_TILE + ko;
                    wgmma_n8(hf[mh], make_desc(al), make_desc(bh), s3);   // small terms first
                    wgmma_n8(hf[mh], make_desc(ah), make_desc(bl), 1);
                    wgmma_n8(hf[mh], make_desc(ah), make_desc(bh), 1);
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            __syncwarp();
            if (lane == 0) mbar_arrive(&phi_empty[st]);
            // ---- activation (the block's own, schnet.py; SFU version of shifted softplus) -> the group's rows of B2
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int ch = mh * 64 + wg_frag_row(c, q), e = wg_frag_col(c, q);
                    const float a = act == SPK_ACT_SSP ? spk_ssp_fast(hf[mh][q]) : spk_act(hf[mh][q], act);
                    const float hi = tf32_rn(a);
                    const int off = tile_off(g * EG + e, (ch & 15) >> 2) + (ch & 3) * 4;
                    *reinterpret_cast<float*>(sB2 + ((ch >> 4) * 2 + 0) * B_TILE + off) = hi;
                    *reinterpret_cast<float*>(sB2 + ((ch >> 4) * 2 + 1) * B_TILE + off) = a - hi;
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            wg_bar(1 + g);
            // ---- MMA 2: D = W1 ssp(H), K = 128
            float dm[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            float dc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
            wgmma_fence();
#pragma unroll
            for (int s16 = 0; s16 < 16; ++s16) {
                const int kt = s16 >> 1, ko = (s16 & 1) * 32;
                const uint32_t bh = bb2 + (kt * 2 + 0) * B_TILE + ko, bl = bb2 + (kt * 2 + 1) * B_TILE + ko;
#pragma unroll
                for (int mh = 0; mh < 2; ++mh) {
                    const uint32_t ah = a1 + (0 * 8 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko;
                    const uint32_t al = a1 + (1 * 8 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko;
                    wgmma_n8(dm[mh], make_desc(ah), make_desc(bh), s16 ? 1 : 0);
                    wgmma_n8(dc[mh], make_desc(al), make_desc(bh), s16 ? 1 : 0);
                    wgmma_n8(dc[mh], make_desc(ah), make_desc(bl), 1);
                }
            }
            wgmma_commit();
            wgmma_wait_all();
            // ---- fragments -> [edge][channel] -> thread = channel
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    tg[wg_frag_col(c, q) * T_LD + mh * 64 + wg_frag_row(c, q)] = dm[mh][q] + dc[mh][q];
            wg_bar(1 + g);
            float w[EG];
#pragma unroll
            for (int u = 0; u < EG; ++u) w[u] = tg[u * T_LD + c];
            mbar_wait(&meta_full[ms], (k / NMETA) & 1);
            const int* st_j = reinterpret_cast<const int*>(sMeta + ms * META_STAGE) + g * EG;
            const float* st_fc = reinterpret_cast<const float*>(sMeta + ms * META_STAGE + NE * 4) + g * EG;
            const int base = s_begin + k * EG;
            if (base < s_end) {
                float hv[EG], fc[EG];
#pragma unroll
                for (int u = 0; u < EG; ++u) {                           // all gathers first (rows past the end read sender 0)
                    hv[u] = h[(size_t)st_j[u] * F + c];
                    fc[u] = st_fc[u];
                }
#pragma unroll
                for (int u = 0; u < EG; ++u) {
                    const int s = base + u;
                    if (s < s_end) {
                        while (s >= next_boundary) {
                            m[(size_t)i * F + c] = acc;
                            acc = 0.f;
                            ++i;
                            next_boundary = rowptr[i + 1];
                        }
                        acc = fmaf((w[u] + b1c) * fc[u], hv[u], acc);
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&meta_empty[ms]);
        }
        for (; i < row_hi; ++i) {
            m[(size_t)i * F + c] = acc;
            acc = 0.f;
        }
    }
}

}  // namespace

extern "C" size_t spk_schnet_filter_packed_floats(void) { return (W0_BYTES + W1_BYTES) / 4; }

extern "C" int spk_schnet_pack_filter(const float* w0, const float* b0, const float* w1, int F, int n_rbf, float* packed,
                                      spk_stream_t stream) {
    if (!w0 || !b0 || !w1 || !packed) return SPK_ERR_ARG;
    if (F != F_TC || n_rbf <= 0 || n_rbf > 31) return SPK_ERR_UNSUPPORTED;
    const int total = F_TC * 32 + F_TC * F_TC;
    spk_launch(k_pack_schnet_filter, (unsigned)spk_cdiv(total, 256), 256, 0, spk_st(stream), w0, b0, w1, n_rbf, packed);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_schnet_cfconv_fwd_tc(const float* h, const float* phi, const float* geo, const int32_t* rowptr,
                                        const int32_t* slot_j, const float* filter_packed, const float* b1, int act,
                                        int64_t n_atoms, int64_t n_edges, int F, int n_rbf, float* m, spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0 || n_rbf <= 0 || act < 0 || act > 2) return SPK_ERR_ARG;
    if (F != F_TC || n_rbf > 31) return SPK_ERR_UNSUPPORTED;
    if (n_atoms == 0) return SPK_OK;
    if (!h || !rowptr || !filter_packed || !m) return SPK_ERR_ARG;
    if (n_edges > 0 && (!phi || !geo || !slot_j)) return SPK_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(phi) | reinterpret_cast<uintptr_t>(filter_packed)) & 15) return SPK_ERR_UNSUPPORTED;
    static SpkSmemOnce once;
    if (cudaError_t e = once.set(k_schnet_cfconv_fwd_tc, SMEM_BYTES); e != cudaSuccess) return SPK_CUDA_ERR(e);
    int64_t nb = spk_num_sms();
    if (nb > spk_cdiv(n_edges, NE) + 1) nb = spk_cdiv(n_edges, NE) + 1;
    if (nb > n_atoms) nb = n_atoms;
    if (nb < 1) nb = 1;
    spk_launch(k_schnet_cfconv_fwd_tc, (unsigned)nb, NTHREADS, SMEM_BYTES, spk_st(stream), h, phi, geo, rowptr, slot_j,
               filter_packed, b1, act, (int)n_atoms, n_rbf, m);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

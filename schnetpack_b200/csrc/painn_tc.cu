// PaiNN fused edge kernel with the continuous filter evaluated on the tensor cores (wgmma).
// Reference: representation/painn.py (message, filter = filter_net(phi) * fcut), nn/scatter.py.
//
// Why: evaluated per channel on the CUDA cores (painn.cu), every warp re-reads the edge's radial-basis values as warp-broadcast
// shared-memory loads to feed its FMAs, and the load/store unit, not HBM, bounds the kernel.  The filter
//       W[e, c] = fc_e * (b_c + sum_k phi_k(d_e) w_ck)            c in [0, 3F)
// is a GEMM with K = n_rbf + 1, so here it runs on the tensor cores instead and the LSU only carries the gathers:
//
//   * orientation: channels on the M side.  For each filter third t the A operand is W_t = [w | b] (128 channels x 32,
//     static, packed once by spk_painn_pack_filter in the shared-memory operand layout and fetched by ONE TMA bulk copy),
//     the B operand is a chunk of 64 edge rows  Phi' = fc * [phi | 1]  (K-major, 64 B swizzle, produced per chunk by
//     the producer warps with the hi/lo split of 3xTF32);
//   * one persistent CTA per SM: 4 consumer warpgroups (a group owns 128 channels of its own edge-balanced receiver range,
//     as a CTA of painn.cu did) and the producer warps.  Group g multiplies W_t by ITS 16 rows of the chunk (wgmma m64n16,
//     two m64 halves), so no group waits for another; the fragments go through a small shared-memory transpose to
//     thread = channel, the mapping of the gather/accumulate code;
//   * 3xTF32 (Wl*Ph + Wh*Pl + Wh*Ph, small terms first) keeps the filter at fp32 accuracy; K = 24 is three k-steps;
//   * NST Phi' stages let the producers stage chunk k+1.. while the groups gather chunk k.
// The reduction over a receiver's edges stays a private register accumulation in CSR order: deterministic, no atomics.
#include "painn_common.cuh"
#include "wgmma.cuh"

#ifdef SPK_EDGE_TRACE                          // -DSPK_EDGE_TRACE=1: forward kernel stamps, =2: reverse kernel stamps
__device__ long long g_edge_trace[SPK_NUM_SMS * 256];
#define EDGE_STAMP(slot)                                                                 \
    do {                                                                                 \
        if ((threadIdx.x & 31) == 0 && (slot) < 256) g_edge_trace[blockIdx.x * 256 + (slot)] = clock64(); \
    } while (0)
extern "C" int spk_debug_edge_trace(long long* host) {
    return (int)cudaMemcpyFromSymbol(host, g_edge_trace, sizeof(long long) * SPK_NUM_SMS * 256);
}
#endif
#if defined(SPK_EDGE_TRACE) && SPK_EDGE_TRACE == 2
#define ETRACE(slot) do { } while (0)
#define BTRACE(slot) EDGE_STAMP(slot)
#elif defined(SPK_EDGE_TRACE)
#define ETRACE(slot) EDGE_STAMP(slot)
#define BTRACE(slot) do { } while (0)
#else
#define ETRACE(slot) do { } while (0)
#define BTRACE(slot) do { } while (0)
#endif

namespace {

constexpr int F_TC = 128;                      // channels per filter third (two m64 halves)
constexpr int EG = 16;                         // edges per group and chunk (wgmma N)
constexpr int NG = 4;                          // consumer groups = warpgroups
constexpr int NE = EG * NG;                    // Phi' rows per chunk
constexpr int NCW = NG * 4;                    // consumer warps
constexpr int W_PROD0 = NCW;
constexpr int NPROD = 3;                       // producer warps: chunk k -> warp k % NPROD
constexpr int NST = 3;                         // Phi' stages: chunk k -> stage k % NST (NPROD divides NST: one owner per stage)
constexpr int NTHREADS = (W_PROD0 + NPROD) * 32;
constexpr int KT = 16;                         // floats per operand K-tile (64 B rows, SWIZZLE_64B)
constexpr int A_TILE = F_TC * KT * 4;          // 8192 B
constexpr int A_BYTES = 3 * 2 * 2 * A_TILE;    // [third][hi,lo][k-tile]
constexpr int B_TILE = NE * KT * 4;            // 4096 B
constexpr int B_STAGE = 2 * 2 * B_TILE;        // [hi,lo][k-tile]
constexpr int META_STAGE = NE * 4 + NE * 16;   // sender index + (ux, uy, uz, -) per row
constexpr int T_LD = F_TC + 4;                 // row of the per-group transpose tile [column][channel] (floats)
constexpr int T_BYTES = NG * 16 * T_LD * 4;    // 16 columns per group (forward: 16 edges; reverse: 8 edges x {W, dW/dd})
constexpr int SMEM_BYTES = A_BYTES + NST * B_STAGE + NST * META_STAGE + T_BYTES + 1024;

// The group's 3xTF32 filter products of one chunk for NT thirds: d[t][m-half] (+)= W_t * B^T over the three k-steps
// (K = n_rbf + 1 <= 24), B = 16 (forward) or 8 (reverse) operand rows starting at byte offset b_row of the stage.
template <int NT, int N>
__device__ __forceinline__ void filter_mma(float (&d)[NT][2][N / 2], uint32_t aB, uint32_t bB) {
    wgmma_fence();
#pragma unroll
    for (int t = 0; t < NT; ++t)
#pragma unroll
        for (int s3 = 0; s3 < 3; ++s3) {                     // k-steps 0..2 = (tile 0, 0), (tile 0, 32 B), (tile 1, 0)
            const int kt = s3 >> 1, ko = (s3 & 1) * 32;
            const uint64_t bh = make_desc(bB + (0 * 2 + kt) * B_TILE + ko);
            const uint64_t bl = make_desc(bB + (1 * 2 + kt) * B_TILE + ko);
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
                const uint64_t ah = make_desc(aB + ((t * 2 + 0) * 2 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko);
                const uint64_t al = make_desc(aB + ((t * 2 + 1) * 2 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko);
                if constexpr (N == 16) {
                    wgmma_n16(d[t][mh], al, bh, s3 ? 1 : 0);       // small terms first
                    wgmma_n16(d[t][mh], ah, bl, 1);
                    wgmma_n16(d[t][mh], ah, bh, 1);
                } else {
                    wgmma_n8(d[t][mh], al, bh, s3 ? 1 : 0);
                    wgmma_n8(d[t][mh], ah, bl, 1);
                    wgmma_n8(d[t][mh], ah, bh, 1);
                }
            }
        }
    wgmma_commit();
    wgmma_wait_all();
}

// fragment (m64nN, two m-halves) of the warpgroup -> columns col0.. of the [column][channel] tile tg
template <int N>
__device__ __forceinline__ void frag_to_tile(const float (&d)[2][N / 2], float* tg, int col0, int t) {
#pragma unroll
    for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) tg[(col0 + wg_frag_col(t, i)) * T_LD + mh * 64 + wg_frag_row(t, i)] = d[mh][i];
}

// [third][hi,lo][k-tile][128 x 16] operand tiles of  [w | b | 0]  (k = n_rbf is the bias column)
__global__ void k_pack_filter(const float* __restrict__ wf, const float* __restrict__ bf, int n_rbf,
                              float* __restrict__ out) {
    SPK_PDL_WAIT_ONLY();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;          // one (third, row, k) element
    if (t >= 3 * F_TC * 32) return;
    const int k = t & 31, row = (t >> 5) % F_TC, third = t / (32 * F_TC);
    const int ch = third * F_TC + row;
    const float w = k < n_rbf ? wf[(int64_t)ch * n_rbf + k] : (k == n_rbf ? bf[ch] : 0.f);
    const float hi = tf32_rn(w), lo = w - hi;
    const int kt = k >> 4, kk = k & 15;
    const int off = tile_off(row, kk >> 2) / 4 + (kk & 3);
    out[((third * 2 + 0) * 2 + kt) * (A_TILE / 4) + off] = hi;
    out[((third * 2 + 1) * 2 + kt) * (A_TILE / 4) + off] = lo;
}

template <bool HAS_MU>
__global__ void __launch_bounds__(NTHREADS, 1) k_painn_edge_fwd_tc(
    const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ q,
    const float* __restrict__ phi, const float* __restrict__ geo, const int* __restrict__ rowptr,
    const int* __restrict__ slot_j, const float* __restrict__ wpk, int n_atoms, int n_edges, int n_rbf,
    float* __restrict__ q_out, float* __restrict__ mu_out) {
    constexpr int F = F_TC;
    constexpr int NT = HAS_MU ? 3 : 2;             // filter thirds in use (mu == 0 makes the third one a no-op)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + A_BYTES;
    uint8_t* sMeta = sB + NST * B_STAGE;
    float* sT = reinterpret_cast<float*>(sMeta + NST * META_STAGE);
    __shared__ __align__(8) uint64_t a_full, full_bar[NST], empty_bar[NST], meta_empty[NST];
    __shared__ int s_rlo[NG], s_rhi[NG], s_sb[NG], s_se[NG];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) ETRACE(0);
    if (tid == 0) {
        mbar_init(&a_full, 1);
#pragma unroll
        for (int s = 0; s < NST; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], NCW);
            mbar_init(&meta_empty[s], NCW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&a_full, A_BYTES);          // static operand: fetched BEFORE griddepcontrol.wait (pack kernels never trigger their dependents early, common.cuh)
        tma_load(sA, wpk, A_BYTES, &a_full);
    }
    SPK_PDL_WAIT();                                // everything below reads memory written by earlier kernels
    if (warp <= NG) {                              // warp w finds boundary w of this CTA's NG group ranges (warp-wide search)
        const int bnd = spk_block_row_begin_warp(rowptr, n_atoms, n_edges, gridDim.x * NG, blockIdx.x * NG + warp);
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
    if (tid == 0) ETRACE(1);

    if (warp >= W_PROD0) {
        // =========================================== producers ===========================================
        const int p = warp - W_PROD0;
        const int qc = lane & 7, rsub = lane >> 3;             // 8 x 16 B K-chunks per row, 4 rows per pass, 16 passes
        const bool q_in = qc * 4 < KP;
        const int kb_chunk = n_rbf >> 2, kb = n_rbf & 3;       // the bias column k = n_rbf
        for (int k = p; k < n_chunks; k += NPROD) {
            const int st = k % NST, use = k / NST;
            uint8_t* stB = sB + st * B_STAGE;
            int* st_j = reinterpret_cast<int*>(sMeta + st * META_STAGE);
            float4* st_u = reinterpret_cast<float4*>(sMeta + st * META_STAGE + NE * 4);
            // all loads are unconditional (rows past a group's end read slot 0 and are zeroed afterwards) and issued in
            // two batches of 8 rows: branchy loads, or more loads than the register budget holds, are serialised by the
            // compiler and cost one full memory latency EACH
            int mj[2];
            float4 mu4[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = lane + 32 * h, g = r / EG;
                const int s = s_sb[g] + k * EG + (r % EG);
                const int sl = s < s_se[g] ? s : 0;
                mj[h] = slot_j[sl];
                mu4[h] = *reinterpret_cast<const float4*>(geo + (int64_t)sl * SPK_GEO_STRIDE);   // ux uy uz d
            }
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float4 pv[8];
                float fcv[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = (half * 8 + i) * 4 + rsub, g = r / EG;
                    const int s = s_sb[g] + k * EG + (r % EG);
                    const bool ok = s < s_se[g];
                    const int sl = ok ? s : 0;
                    const float fc = geo[(int64_t)sl * SPK_GEO_STRIDE + 4];
                    fcv[i] = ok ? fc : 0.f;
                    pv[i] = *reinterpret_cast<const float4*>(phi + (int64_t)sl * KP + (q_in ? qc * 4 : 0));
                }
                if (half == 0) {
                    if (p == 0 && k < 48) ETRACE(16 + k / 3);  // producer 0: loads issued
                    if (use >= 1) {
                        mbar_wait(&empty_bar[st], (use - 1) & 1);      // MMAs of chunk k-NST have read this Phi' stage
                        mbar_wait(&meta_empty[st], (use - 1) & 1);     // consumers are done with its metadata
                    }
                }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int r = (half * 8 + i) * 4 + rsub;
                    const float fc = fcv[i];                   // 0 for rows past the group's end
                    float4 v = q_in ? pv[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (qc == kb_chunk) {
                        if (kb == 0) v.x = 1.f; else if (kb == 1) v.y = 1.f; else if (kb == 2) v.z = 1.f; else v.w = 1.f;
                    }
                    v.x *= fc; v.y *= fc; v.z *= fc; v.w *= fc;  // Phi' = fc * [phi | 1]: the MMA yields W itself
                    float4 hi, lo;
                    hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
                    lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
                    const int off = tile_off(r, qc & 3);
                    *reinterpret_cast<float4*>(stB + (0 * 2 + (qc >> 2)) * B_TILE + off) = hi;
                    *reinterpret_cast<float4*>(stB + (1 * 2 + (qc >> 2)) * B_TILE + off) = lo;
                }
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                st_j[lane + 32 * h] = mj[h];
                st_u[lane + 32 * h] = mu4[h];
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[st]);
            if (p == 0 && k < 48) ETRACE(32 + k / 3);          // producer 0: published
        }
    } else {
        // =========================================== consumers ===========================================
        const int g = warp >> 2, qd = warp & 3;
        const int c = qd * 32 + lane;                          // channel (thread of the warpgroup)
        const int row_hi = s_rhi[g], s_begin = s_sb[g], s_end = s_se[g];
        int i = s_rlo[g];
        int next_boundary = i < row_hi ? rowptr[i + 1] : 0x7fffffff;
        float dq = 0.f, dm0 = 0.f, dm1 = 0.f, dm2 = 0.f;
        // The residual inputs of the CURRENT receiver row and the row pointer after next are fetched when the row starts,
        // not when it ends: a row switch then costs four stores instead of two dependent memory latencies (row pointer ->
        // q / mu rows -> stores) in front of the next edge.
        float bq = 0.f, bm0 = 0.f, bm1 = 0.f, bm2 = 0.f;
        int boundary2 = 0x7fffffff;
        auto prefetch_row = [&](int row) {                     // row <= row_hi <= n_atoms; clamped reads are never used
            const int r = row < n_atoms ? row : n_atoms - 1;
            boundary2 = rowptr[min(row + 2, n_atoms)];
            bq = q[(size_t)r * F + c];
            if (HAS_MU) {
                const float* __restrict__ mr = mu + (size_t)r * 3 * F + c;
                bm0 = mr[0];
                bm1 = mr[F];
                bm2 = mr[2 * F];
            }
        };
        prefetch_row(i);
        auto flush = [&](int row) {                            // row == i: its residual inputs are in bq / bm*
            q_out[(size_t)row * F + c] = bq + dq;
            const size_t om = (size_t)row * 3 * F + c;
            mu_out[om] = bm0 + dm0;
            mu_out[om + F] = bm1 + dm1;
            mu_out[om + 2 * F] = bm2 + dm2;
            dq = dm0 = dm1 = dm2 = 0.f;
        };
        float* tg = sT + g * 16 * T_LD;                        // this group's [edge][channel] transpose tile
        const uint32_t aB = smem_u32(sA);
        mbar_wait(&a_full, 0);
        for (int k = 0; k < n_chunks; ++k) {
            const int st = k % NST;
            if (warp == 0 && k < 16) ETRACE(64 + k);           // consumer 0: starts waiting
            mbar_wait(&full_bar[st], (k / NST) & 1);           // Phi' rows and metadata of the chunk
            float d[NT][2][8];
            filter_mma<NT, 16>(d, aB, smem_u32(sB + st * B_STAGE) + (uint32_t)(g * EG * SPK_SW64_ROW));
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[st]);        // the group's wgmma have read the stage
            float wv[3][EG];
#pragma unroll
            for (int t = 0; t < NT; ++t) {                     // fragments -> thread = channel, one third at a time
                frag_to_tile<16>(d[t], tg, 0, c);
                wg_bar(1 + g);
#pragma unroll
                for (int u = 0; u < EG; ++u) wv[t][u] = tg[u * T_LD + c];
                wg_bar(1 + g);
            }
            if (warp == 0 && k < 16) ETRACE(80 + k);           // filter values ready
            if (warp == 0 && lane == 0 && k == 0) SPK_TL_PHASE(2);
            const int* st_j = reinterpret_cast<const int*>(sMeta + st * META_STAGE) + g * EG;
            const float4* st_u = reinterpret_cast<const float4*>(sMeta + st * META_STAGE + NE * 4) + g * EG;
            const int base = s_begin + k * EG;
            // eight edges at a time: all their gathers are issued before the first use (rows past the range read sender 0,
            // their filter values are exactly 0), so eight memory latencies overlap instead of following each other
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                constexpr int HB = EG / 2;
                const float* wa = wv[0] + half * HB;
                const float* wb = wv[1] + half * HB;
                const float* wc = wv[2] + half * HB;
                if (base + half * HB < s_end) {
                    float xa[HB], xb[HB], xc[HB], m0[HB], m1[HB], m2[HB];
#pragma unroll
                    for (int u = 0; u < HB; ++u) {
#ifdef SPK_EDGE_EXP_JMASK
                        const int j = st_j[half * HB + u] & 7;     // experiment: all gathers hit L1 (timing only)
#else
                        const int j = st_j[half * HB + u];
#endif
                        const float* __restrict__ xj = x + (size_t)j * (3 * F) + c;
                        xa[u] = xj[0];
                        xb[u] = xj[F];
                        if (HAS_MU) {
                            xc[u] = xj[2 * F];
                            const float* __restrict__ mj = mu + (size_t)j * (3 * F) + c;
                            m0[u] = mj[0];
                            m1[u] = mj[F];
                            m2[u] = mj[2 * F];
                        }
                    }
#pragma unroll
                    for (int u = 0; u < HB; ++u) {
                        const int t = half * HB + u;
                        const int s = base + t;
                        if (s < s_end) {
                            while (s >= next_boundary) {
                                flush(i);
                                ++i;
                                next_boundary = boundary2;
                                prefetch_row(i);
                            }
                            const float4 uv = st_u[t];
                            dq = fmaf(wa[u], xa[u], dq);
                            const float tb = wb[u] * xb[u];
                            dm0 = fmaf(tb, uv.x, dm0);
                            dm1 = fmaf(tb, uv.y, dm1);
                            dm2 = fmaf(tb, uv.z, dm2);
                            if (HAS_MU) {
                                const float tc = wc[u] * xc[u];
                                dm0 = fmaf(tc, m0[u], dm0);
                                dm1 = fmaf(tc, m1[u], dm1);
                                dm2 = fmaf(tc, m2[u], dm2);
                            }
                        }
                    }
                }
                if (half == 0 && warp == 0 && k < 16) ETRACE(128 + k);     // first half's edges done
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&meta_empty[st]);
            if (warp == 0 && k < 16) ETRACE(96 + k);           // chunk's edges done
        }
        if (warp == 0) ETRACE(2);
        if (warp == 0 && lane == 0) SPK_TL_PHASE(3);           // main loop done
        for (; i < row_hi;) {
            flush(i);
            ++i;
            prefetch_row(i);
        }
        if (warp == 0) ETRACE(3);
    }
}


// ------------------------------------------------------------------------------------------------------------------
// reverse pass, grouped by sender (same structure; reference: autograd of painn.py:55-65)
// ------------------------------------------------------------------------------------------------------------------
// A chunk is 4 groups x 8 edges.  Its operand has 64 rows: rows 0..31 = fc [phi | 1] (-> W) and rows 32..63 =
// dfc [phi | 1] + fc [dphi | 0] (-> dW/dd); group g multiplies its 8 rows of each half, so one pass yields both the filter
// and its radial derivative.
constexpr int EGB = 8;                         // edges per group and chunk
constexpr int NEB = EGB * NG;                  // 32 edges per chunk (x 2 operand rows each)
constexpr int META_B = NEB * 4 + NEB * 4 + NEB * 16;   // receiver index, edge id, (ux, uy, uz, 1/d) per edge
constexpr int SMEM_BYTES_B = A_BYTES + NST * B_STAGE + NST * META_B + T_BYTES + 1024;


template <bool HAS_MU>
__global__ void __launch_bounds__(NTHREADS, 1) k_painn_edge_bwd_tc(
    const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ g_q,
    const float* __restrict__ g_mu, const float* __restrict__ phi, const float* __restrict__ dphi,
    const float* __restrict__ geo, const int* __restrict__ sptr, const int* __restrict__ pos_slot,
    const int* __restrict__ pos_i, const int* __restrict__ slot_eid, const float* __restrict__ wpk, int n_atoms,
    int n_edges, int n_rbf, float* __restrict__ g_x, float* __restrict__ g_mu_in, float* __restrict__ g_rij,
    int accumulate) {
    constexpr int F = F_TC;
    constexpr int NT = HAS_MU ? 3 : 2;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA = smem;
    uint8_t* sB = smem + A_BYTES;
    uint8_t* sMeta = sB + NST * B_STAGE;
    float* sT = reinterpret_cast<float*>(sMeta + NST * META_B);
    __shared__ __align__(8) uint64_t a_full, full_bar[NST], empty_bar[NST], meta_empty[NST];
    __shared__ int s_rlo[NG], s_rhi[NG], s_sb[NG], s_se[NG];
    __shared__ float s_red[2][NG][EGB][4][4];      // [chunk parity][group][edge][warp][scalar]

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) {
        mbar_init(&a_full, 1);
#pragma unroll
        for (int s = 0; s < NST; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], NCW);
            mbar_init(&meta_empty[s], NCW);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&a_full, A_BYTES);          // static operand: fetched BEFORE griddepcontrol.wait (pack kernels never trigger their dependents early, common.cuh)
        tma_load(sA, wpk, A_BYTES, &a_full);
    }
    if (tid == 0) BTRACE(0);
    SPK_PDL_WAIT();
    if (tid == 0) BTRACE(1);
    if (warp <= NG) {                              // warp w finds boundary w of this CTA's NG group ranges (warp-wide search)
        const int bnd = spk_block_row_begin_warp(sptr, n_atoms, n_edges, gridDim.x * NG, blockIdx.x * NG + warp);
        if (lane == 0) {
            const int e = sptr[bnd];
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
    for (int g = 0; g < NG; ++g) n_chunks = max(n_chunks, (s_se[g] - s_sb[g] + EGB - 1) / EGB);
    const int KP = spk_kp(n_rbf);

    if (warp >= W_PROD0) {
        // =========================================== producers ===========================================
        const int p = warp - W_PROD0;
        const int qc = lane & 7, rsub = lane >> 3;             // 8 x 16 B K-chunks per row, 4 edges per pass, 8 passes
        const bool q_in = qc * 4 < KP;
        const int kb_chunk = n_rbf >> 2, kb = n_rbf & 3;
        for (int k = p; k < n_chunks; k += NPROD) {
            const int st = k % NST, use = k / NST;
            uint8_t* stB = sB + st * B_STAGE;
            int* st_i = reinterpret_cast<int*>(sMeta + st * META_B);
            int* st_e = st_i + NEB;
            float4* st_u = reinterpret_cast<float4*>(sMeta + st * META_B + 2 * NEB * 4);
            // consumer metadata: lane = edge of the chunk
            int m_i, m_e;
            float4 m_u;
            {
                const int g = lane / EGB;
                const int pp = s_sb[g] + k * EGB + (lane % EGB);
                const bool ok = pp < s_se[g];
                const int sl = pos_slot[ok ? pp : 0];
                m_i = pos_i[ok ? pp : 0];
                m_e = slot_eid[sl];
                const float4 g0 = *reinterpret_cast<const float4*>(geo + (int64_t)sl * SPK_GEO_STRIDE);
                m_u = make_float4(g0.x, g0.y, g0.z, geo[(int64_t)sl * SPK_GEO_STRIDE + 6]);
            }
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                float4 pv[4], dv[4];
                float fcv[4], dfcv[4];
                int sl[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = (half * 4 + i) * 4 + rsub, g = r / EGB;
                    const int pp = s_sb[g] + k * EGB + (r % EGB);
                    const bool ok = pp < s_se[g];
                    sl[i] = pos_slot[ok ? pp : 0];
                    fcv[i] = ok ? 1.f : 0.f;
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f2 = *reinterpret_cast<const float2*>(geo + (int64_t)sl[i] * SPK_GEO_STRIDE + 4);   // fc, dfc
                    dfcv[i] = f2.y * fcv[i];
                    fcv[i] *= f2.x;
                    pv[i] = *reinterpret_cast<const float4*>(phi + (int64_t)sl[i] * KP + (q_in ? qc * 4 : 0));
                    dv[i] = *reinterpret_cast<const float4*>(dphi + (int64_t)sl[i] * KP + (q_in ? qc * 4 : 0));
                }
                if (half == 0 && use >= 1) {
                    mbar_wait(&empty_bar[st], (use - 1) & 1);
                    mbar_wait(&meta_empty[st], (use - 1) & 1);
                }
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int r = (half * 4 + i) * 4 + rsub;
                    const float fc = fcv[i], dfc = dfcv[i];
                    float4 v = q_in ? pv[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                    float4 d = q_in ? dv[i] : make_float4(0.f, 0.f, 0.f, 0.f);
                    if (qc == kb_chunk) {                      // bias column: [phi | 1], [dphi | 0]
                        if (kb == 0) { v.x = 1.f; d.x = 0.f; } else if (kb == 1) { v.y = 1.f; d.y = 0.f; }
                        else if (kb == 2) { v.z = 1.f; d.z = 0.f; } else { v.w = 1.f; d.w = 0.f; }
                    }
                    float4 w, dw;                              // rows of the W and dW/dd operands
                    w.x = fc * v.x; w.y = fc * v.y; w.z = fc * v.z; w.w = fc * v.w;
                    dw.x = fmaf(dfc, v.x, fc * d.x); dw.y = fmaf(dfc, v.y, fc * d.y);
                    dw.z = fmaf(dfc, v.z, fc * d.z); dw.w = fmaf(dfc, v.w, fc * d.w);
                    float4 hi, lo;
                    hi.x = tf32_rn(w.x); hi.y = tf32_rn(w.y); hi.z = tf32_rn(w.z); hi.w = tf32_rn(w.w);
                    lo.x = w.x - hi.x; lo.y = w.y - hi.y; lo.z = w.z - hi.z; lo.w = w.w - hi.w;
                    int off = tile_off(r, qc & 3);
                    *reinterpret_cast<float4*>(stB + (0 * 2 + (qc >> 2)) * B_TILE + off) = hi;
                    *reinterpret_cast<float4*>(stB + (1 * 2 + (qc >> 2)) * B_TILE + off) = lo;
                    hi.x = tf32_rn(dw.x); hi.y = tf32_rn(dw.y); hi.z = tf32_rn(dw.z); hi.w = tf32_rn(dw.w);
                    lo.x = dw.x - hi.x; lo.y = dw.y - hi.y; lo.z = dw.z - hi.z; lo.w = dw.w - hi.w;
                    off = tile_off(NEB + r, qc & 3);
                    *reinterpret_cast<float4*>(stB + (0 * 2 + (qc >> 2)) * B_TILE + off) = hi;
                    *reinterpret_cast<float4*>(stB + (1 * 2 + (qc >> 2)) * B_TILE + off) = lo;
                }
            }
            st_i[lane] = m_i;
            st_e[lane] = m_e;
            st_u[lane] = m_u;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[st]);
        }
    } else {
        // =========================================== consumers ===========================================
        const int g = warp >> 2, qd = warp & 3;
        const int c = qd * 32 + lane;
        const int j_hi = s_rhi[g], p_begin = s_sb[g], p_end = s_se[g];
        int j = s_rlo[g];
        int next_boundary = j < j_hi ? sptr[j + 1] : 0x7fffffff;
        float xa = 0.f, xb = 0.f, xc = 0.f, m0 = 0.f, m1 = 0.f, m2 = 0.f;
        float gxa = 0.f, gxb = 0.f, gxc = 0.f, gm0 = 0.f, gm1 = 0.f, gm2 = 0.f;
        auto load_own = [&](int row) {
            const float* __restrict__ xr = x + (size_t)row * (3 * F) + c;
            xa = xr[0];
            xb = xr[F];
            if (HAS_MU) {
                xc = xr[2 * F];
                const float* __restrict__ mr = mu + (size_t)row * (3 * F) + c;
                m0 = mr[0];
                m1 = mr[F];
                m2 = mr[2 * F];
            }
        };
        auto flush = [&](int row) {
            const size_t o = (size_t)row * 3 * F + c;
            g_x[o] = gxa;
            g_x[o + F] = gxb;
            g_x[o + 2 * F] = gxc;
            if (HAS_MU) {
                g_mu_in[o] = g_mu[o] + gm0;
                g_mu_in[o + F] = g_mu[o + F] + gm1;
                g_mu_in[o + 2 * F] = g_mu[o + 2 * F] + gm2;
            }
            gxa = gxb = gxc = gm0 = gm1 = gm2 = 0.f;
        };
        if (j < j_hi) load_own(j);
        const int my_idx = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
        float* tg = sT + g * 16 * T_LD;                        // this group's [W edge | dW edge][channel] transpose tile
        const uint32_t aB = smem_u32(sA);
        mbar_wait(&a_full, 0);
        for (int k = 0; k < n_chunks; ++k) {
            const int st = k % NST;
            if (warp == 0 && k < 16) BTRACE(64 + k);           // consumer 0: starts waiting
            mbar_wait(&full_bar[st], (k / NST) & 1);           // operand rows and metadata of the chunk
            const uint32_t bB = smem_u32(sB + st * B_STAGE);
            float dw[NT][2][4], dd[NT][2][4];
            filter_mma<NT, 8>(dw, aB, bB + (uint32_t)(g * EGB * SPK_SW64_ROW));           // W rows of the group
            filter_mma<NT, 8>(dd, aB, bB + (uint32_t)((NEB + g * EGB) * SPK_SW64_ROW));   // dW/dd rows of the group
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[st]);
            float wv[3][EGB], dv[3][EGB];
#pragma unroll
            for (int t = 0; t < NT; ++t) {                     // fragments -> thread = channel, one third at a time
                frag_to_tile<8>(dw[t], tg, 0, c);
                frag_to_tile<8>(dd[t], tg, EGB, c);
                wg_bar(1 + g);
#pragma unroll
                for (int u = 0; u < EGB; ++u) {
                    wv[t][u] = tg[u * T_LD + c];
                    dv[t][u] = tg[(EGB + u) * T_LD + c];
                }
                wg_bar(1 + g);
            }
            if (warp == 0 && k < 16) BTRACE(80 + k);           // filter values + metadata ready
            if (warp == 0 && lane == 0 && k == 0) SPK_TL_PHASE(2);
            const int* st_i = reinterpret_cast<const int*>(sMeta + st * META_B) + g * EGB;
            const int* st_e = reinterpret_cast<const int*>(sMeta + st * META_B) + NEB + g * EGB;
            const float4* st_u = reinterpret_cast<const float4*>(sMeta + st * META_B + 2 * NEB * 4) + g * EGB;
            const int base = p_begin + k * EGB;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const float *Wa = wv[0] + half * 4, *Wb = wv[1] + half * 4, *Wc = wv[2] + half * 4;
                const float *Da = dv[0] + half * 4, *Db = dv[1] + half * 4, *Dc = dv[2] + half * 4;
                float gq[4], g0[4], g1[4], g2[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {                  // rows past the range gather receiver 0; their W, dW are 0
                    const int i = st_i[half * 4 + u];
                    gq[u] = g_q[(size_t)i * F + c];
                    const float* __restrict__ gmi = g_mu + (size_t)i * (3 * F) + c;
                    g0[u] = gmi[0];
                    g1[u] = gmi[F];
                    g2[u] = gmi[2 * F];
                }
                float red[16];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int t = half * 4 + u;
                    const int p = base + t;
                    float part_d = 0.f, pu0 = 0.f, pu1 = 0.f, pu2 = 0.f;
                    if (p < p_end) {
                        if (p >= next_boundary) {
                            do {
                                flush(j);
                                ++j;
                                next_boundary = sptr[j + 1];
                            } while (p >= next_boundary);
                            load_own(j);
                        }
                        const float4 ge = st_u[t];                 // ux uy uz 1/d
                        const float gu = g0[u] * ge.x + g1[u] * ge.y + g2[u] * ge.z;
                        gxa = fmaf(Wa[u], gq[u], gxa);
                        gxb = fmaf(Wb[u], gu, gxb);
                        part_d = gq[u] * xa * Da[u] + gu * xb * Db[u];
                        const float wbx = Wb[u] * xb;
                        pu0 = g0[u] * wbx;
                        pu1 = g1[u] * wbx;
                        pu2 = g2[u] * wbx;
                        if (HAS_MU) {
                            const float gm = g0[u] * m0 + g1[u] * m1 + g2[u] * m2;
                            gxc = fmaf(Wc[u], gm, gxc);
                            const float wcx = Wc[u] * xc;
                            gm0 = fmaf(wcx, g0[u], gm0);
                            gm1 = fmaf(wcx, g1[u], gm1);
                            gm2 = fmaf(wcx, g2[u], gm2);
                            part_d = fmaf(gm * xc, Dc[u], part_d);
                        }
                    }
                    red[4 * u + 0] = part_d;
                    red[4 * u + 1] = pu0;
                    red[4 * u + 2] = pu1;
                    red[4 * u + 3] = pu2;
                }
                const float tot = butterfly16(red, lane);
                const int te = half * 4 + (my_idx >> 2);
                if (!(lane & 1)) s_red[k & 1][g][te][qd][my_idx & 3] = tot;
                if (warp == 0 && k < 16) BTRACE((half ? 128 : 112) + k);   // half done (4 edges + butterfly)
            }
            // the four warps of the group have published their partial sums of this chunk's 8 edges
            asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
            if (warp == 0 && k < 16) BTRACE(144 + k);          // group barrier passed
            if (qd == 0 && lane < EGB && base + lane < p_end) {
                const int t = lane;
                float gd = 0.f, u0 = 0.f, u1 = 0.f, u2 = 0.f;
#pragma unroll
                for (int wv = 0; wv < 4; ++wv) {
                    gd += s_red[k & 1][g][t][wv][0];
                    u0 += s_red[k & 1][g][t][wv][1];
                    u1 += s_red[k & 1][g][t][wv][2];
                    u2 += s_red[k & 1][g][t][wv][3];
                }
                const float4 ge = st_u[t];
                const float dot = u0 * ge.x + u1 * ge.y + u2 * ge.z;
                float r0 = gd * ge.x + (u0 - dot * ge.x) * ge.w;
                float r1 = gd * ge.y + (u1 - dot * ge.y) * ge.w;
                float r2 = gd * ge.z + (u2 - dot * ge.z) * ge.w;
                float* out = g_rij + (int64_t)st_e[t] * 3;
                if (accumulate) {
                    r0 += out[0];
                    r1 += out[1];
                    r2 += out[2];
                }
                out[0] = r0;
                out[1] = r1;
                out[2] = r2;
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&meta_empty[st]);
            if (warp == 0 && k < 16) BTRACE(96 + k);           // chunk done (incl. the g_rij tail of warp qd == 0)
        }
        if (warp == 0 && lane == 0) SPK_TL_PHASE(3);           // main loop done
        if (warp == 0) BTRACE(2);
        for (; j < j_hi; ++j) flush(j);
        if (warp == 0) BTRACE(3);
    }
}

}  // namespace

extern "C" size_t spk_painn_filter_packed_floats(void) { return (size_t)A_BYTES / 4; }

extern "C" int spk_painn_pack_filter(const float* wf, const float* bf, int F, int n_rbf, float* packed,
                                     spk_stream_t stream) {
    if (!wf || !bf || !packed) return SPK_ERR_ARG;
    if (F != F_TC || n_rbf <= 0 || n_rbf > 31) return SPK_ERR_UNSUPPORTED;
    spk_launch(k_pack_filter, (unsigned)spk_cdiv(3 * F_TC * 32, 256), 256, 0, spk_st(stream), wf, bf, n_rbf, packed);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_edge_fwd_tc(const float* x, const float* mu, const float* q, const float* phi, const float* geo,
                                     const int32_t* rowptr, const int32_t* slot_j, const float* wf_packed,
                                     int64_t n_atoms, int64_t n_edges, int F, int n_rbf, float* q_out, float* mu_out,
                                     spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (F != F_TC || n_rbf > 31 || n_edges == 0) return SPK_ERR_UNSUPPORTED;      // caller uses spk_painn_edge_fwd
    if (n_atoms == 0) return SPK_OK;
    if (!x || !q || !phi || !geo || !rowptr || !slot_j || !wf_packed || !q_out || !mu_out) return SPK_ERR_ARG;
    if (mu && mu == mu_out) return SPK_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(phi) | reinterpret_cast<uintptr_t>(geo) | reinterpret_cast<uintptr_t>(wf_packed)) & 15)
        return SPK_ERR_UNSUPPORTED;
    static SpkSmemOnce once_mu, once_nomu;
    if (cudaError_t e = once_mu.set(k_painn_edge_fwd_tc<true>, SMEM_BYTES); e != cudaSuccess) return SPK_CUDA_ERR(e);
    if (cudaError_t e = once_nomu.set(k_painn_edge_fwd_tc<false>, SMEM_BYTES); e != cudaSuccess) return SPK_CUDA_ERR(e);
    int64_t nb = spk_num_sms();
    if (nb > spk_cdiv(n_edges, NE)) nb = spk_cdiv(n_edges, NE);
    if (nb > n_atoms) nb = n_atoms;
    if (nb < 1) nb = 1;
    cudaStream_t st = spk_st(stream);
    if (mu)
        spk_launch(k_painn_edge_fwd_tc<true>, (unsigned)nb, NTHREADS, SMEM_BYTES, st, x, mu, q, phi, geo, rowptr, slot_j,
                   wf_packed, (int)n_atoms, (int)n_edges, n_rbf, q_out, mu_out);
    else
        spk_launch(k_painn_edge_fwd_tc<false>, (unsigned)nb, NTHREADS, SMEM_BYTES, st, x, mu, q, phi, geo, rowptr, slot_j,
                   wf_packed, (int)n_atoms, (int)n_edges, n_rbf, q_out, mu_out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_edge_bwd_tc(const float* x, const float* mu, const float* g_q, const float* g_mu,
                                     const float* phi, const float* dphi, const float* geo, const int32_t* sptr,
                                     const int32_t* pos_slot, const int32_t* pos_i, const int32_t* slot_eid,
                                     const float* wf_packed, int64_t n_atoms, int64_t n_edges, int F, int n_rbf,
                                     float* g_x, float* g_mu_in, float* g_rij, int accumulate, spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (F != F_TC || n_rbf > 31 || n_edges == 0) return SPK_ERR_UNSUPPORTED;      // caller uses spk_painn_edge_bwd
    if (n_atoms == 0) return SPK_OK;
    if (!x || !g_q || !g_mu || !phi || !dphi || !geo || !sptr || !pos_slot || !pos_i || !slot_eid || !wf_packed || !g_x ||
        !g_rij)
        return SPK_ERR_ARG;
    if (mu && !g_mu_in) return SPK_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(phi) | reinterpret_cast<uintptr_t>(dphi) | reinterpret_cast<uintptr_t>(geo) |
         reinterpret_cast<uintptr_t>(wf_packed)) & 15)
        return SPK_ERR_UNSUPPORTED;
    static SpkSmemOnce once_mu, once_nomu;
    if (cudaError_t e = once_mu.set(k_painn_edge_bwd_tc<true>, SMEM_BYTES_B); e != cudaSuccess) return SPK_CUDA_ERR(e);
    if (cudaError_t e = once_nomu.set(k_painn_edge_bwd_tc<false>, SMEM_BYTES_B); e != cudaSuccess) return SPK_CUDA_ERR(e);
    int64_t nb = spk_num_sms();
    if (nb > spk_cdiv(n_edges, NEB)) nb = spk_cdiv(n_edges, NEB);
    if (nb > n_atoms) nb = n_atoms;
    if (nb < 1) nb = 1;
    cudaStream_t st = spk_st(stream);
    if (mu)
        spk_launch(k_painn_edge_bwd_tc<true>, (unsigned)nb, NTHREADS, SMEM_BYTES_B, st, x, mu, g_q, g_mu, phi, dphi, geo, sptr,
                   pos_slot, pos_i, slot_eid, wf_packed, (int)n_atoms, (int)n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate);
    else
        spk_launch(k_painn_edge_bwd_tc<false>, (unsigned)nb, NTHREADS, SMEM_BYTES_B, st, x, mu, g_q, g_mu, phi, dphi, geo, sptr,
                   pos_slot, pos_i, slot_eid, wf_packed, (int)n_atoms, (int)n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

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
//     the B operand is a chunk of NR = 32 operand rows  Phi' = fc * [phi | 1]  (K-major, 64 B swizzle, hi/lo split of 3xTF32);
//   * one persistent CTA per SM: 4 consumer warpgroups (a group owns 128 channels of its own edge-balanced receiver range,
//     as a CTA of painn.cu did) and one producer warpgroup.  The producer stages the Phi' rows of a whole chunk (every
//     group's rows), multiplies them with wide wgmma (m64n32k8: 3 thirds x 2 m-halves x 3 k-steps x 3 products = 54
//     instructions per chunk) and stores the fragments straight into a [operand row][third * 128 + channel] fp32 tile;
//     the consumers read their rows of it with thread = channel, the mapping of the gather/accumulate code.  They never
//     issue or wait on a wgmma, so the tensor core and the gathers run side by side;
//   * 3xTF32 (Wl*Ph + Wh*Pl + Wh*Ph, small terms first) keeps the filter at fp32 accuracy; K = 24 is three k-steps;
//   * NBUF = 2 filter tiles (with their metadata) behind full/empty mbarriers: the producer stages, multiplies and stores
//     chunk k+1 while the groups gather chunk k.  The global loads of chunk k+1 are issued before the MMAs of chunk k and
//     land while they run.
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
// Stamp slots (consumer warp 0, chunks k < 16): 64+k the wait for the chunk starts, 176+k it returns, 80+k the filter
// values are in registers, 96+k the chunk is done; 16+k (producer warp 0): the chunk's filter tile is published.

namespace {

constexpr int F_TC = 128;                      // channels per filter third (two m64 halves)
constexpr int NG = 4;                          // consumer groups = warpgroups
constexpr int NCW = NG * 4;                    // consumer warps
constexpr int W_PROD0 = NCW;                   // the producer warpgroup: warps NCW .. NCW + 3
constexpr int NTHREADS = (NCW + 4) * 32;
constexpr int PROD_BAR = 1 + NG;               // named barrier of the producer warpgroup (1..NG: consumer groups)
constexpr int NR = 32;                         // operand rows per chunk = wgmma N
constexpr int NBUF = 2;                        // filter tiles (and their metadata) in flight
constexpr int KT = 16;                         // floats per operand K-tile (64 B rows, SWIZZLE_64B)
constexpr int A_TILE = F_TC * KT * 4;          // 8192 B
constexpr int A_BYTES = 3 * 2 * 2 * A_TILE;    // [third][hi,lo][k-tile]
constexpr int B_TILE = NR * KT * 4;            // 2048 B
constexpr int B_BYTES = 2 * 2 * B_TILE;        // [hi,lo][k-tile]
constexpr int T_LD = 3 * F_TC + 4;             // row of the filter tile (floats); = 4 mod 32: conflict-free fragment stores
constexpr int T_FLOATS = NR * T_LD;
constexpr int T_BYTES = T_FLOATS * 4;

// Forward: a chunk is NG groups x EG edges, one operand row each.
constexpr int EG = NR / NG;                    // 8 edges per group and chunk
constexpr int META_F = NR * 4 + NR * 16;       // sender index + (ux, uy, uz, -) per row
constexpr int SMEM_BYTES = A_BYTES + B_BYTES + NBUF * (T_BYTES + META_F) + 1024;

// One filter third on the producer warpgroup: d[m-half] = W_t * B^T over the three k-steps (K = n_rbf + 1 <= 24) for the
// NR operand rows of the stage at bB, as one commit group.
__device__ __forceinline__ void filter_third(float (&d)[2][16], uint32_t aB, uint32_t bB, int t) {
    wgmma_fence();
#pragma unroll
    for (int s3 = 0; s3 < 3; ++s3) {                         // k-steps 0..2 = (tile 0, 0), (tile 0, 32 B), (tile 1, 0)
        const int kt = s3 >> 1, ko = (s3 & 1) * 32;
        const uint64_t bh = make_desc(bB + (0 * 2 + kt) * B_TILE + ko);
        const uint64_t bl = make_desc(bB + (1 * 2 + kt) * B_TILE + ko);
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
            const uint64_t ah = make_desc(aB + ((t * 2 + 0) * 2 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko);
            const uint64_t al = make_desc(aB + ((t * 2 + 1) * 2 + kt) * A_TILE + mh * SPK_WG_ROWS_BYTES + ko);
            wgmma_n32(d[mh], al, bh, s3 ? 1 : 0);              // small terms first
            wgmma_n32(d[mh], ah, bl, 1);
            wgmma_n32(d[mh], ah, bh, 1);
        }
    }
    wgmma_commit();
}

// The chunk's 3xTF32 filter for NT thirds -> tile[row][t * 128 + channel].  Third t+1 is on the tensor core while the
// fragments of third t are stored (pt: thread of the producer warpgroup).
template <int NT>
__device__ __forceinline__ void filter_to_tile(uint32_t aB, uint32_t bB, float* tile, int pt) {
    float d[2][2][16];                                       // [third parity][m-half]
    filter_third(d[0], aB, bB, 0);
#pragma unroll
    for (int t = 0; t < NT; ++t) {
        if (t + 1 < NT) {
            filter_third(d[(t + 1) & 1], aB, bB, t + 1);
            wgmma_wait<1>();
        } else {
            wgmma_wait<0>();
        }
#pragma unroll
        for (int mh = 0; mh < 2; ++mh)
#pragma unroll
            for (int i = 0; i < 16; ++i)
                tile[wg_frag_col(pt, i) * T_LD + t * F_TC + mh * 64 + wg_frag_row(pt, i)] = d[t & 1][mh][i];
    }
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

// 16-byte chunk of one Phi' row -> the hi/lo operand tiles of the stage
__device__ __forceinline__ void put_row(uint8_t* stB, int r, int qc, float4 v) {
    float4 hi, lo;
    hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
    lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
    const int off = tile_off(r, qc & 3);
    *reinterpret_cast<float4*>(stB + (0 * 2 + (qc >> 2)) * B_TILE + off) = hi;
    *reinterpret_cast<float4*>(stB + (1 * 2 + (qc >> 2)) * B_TILE + off) = lo;
}

// [phi | 1] restricted to the 16-byte K-chunk qc (the bias column k = n_rbf is 1, chunks past KP are 0)
__device__ __forceinline__ float4 with_bias(float4 v, bool q_in, int qc, int n_rbf) {
    if (!q_in) v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (qc == (n_rbf >> 2)) {
        const int kb = n_rbf & 3;
        if (kb == 0) v.x = 1.f; else if (kb == 1) v.y = 1.f; else if (kb == 2) v.z = 1.f; else v.w = 1.f;
    }
    return v;
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
    float* sT = reinterpret_cast<float*>(sB + B_BYTES);
    uint8_t* sMeta = sB + B_BYTES + NBUF * T_BYTES;
    __shared__ __align__(8) uint64_t a_full, full_bar[NBUF], empty_bar[NBUF];
    __shared__ int s_rlo[NG], s_rhi[NG], s_sb[NG], s_se[NG];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) ETRACE(0);
    if (tid == 0) {
        mbar_init(&a_full, 1);
#pragma unroll
        for (int b = 0; b < NBUF; ++b) {
            mbar_init(&full_bar[b], 4);
            mbar_init(&empty_bar[b], NCW);
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
        const int pt = tid - W_PROD0 * 32;                     // thread of the producer warpgroup
        const int qc = pt & 7, rsub = pt >> 3;                 // 8 x 16 B K-chunks per row, 16 rows per pass, 2 passes
        const bool q_in = qc * 4 < KP;
        // one chunk in registers: all loads are unconditional (rows past a group's end read slot 0, fc = 0 zeroes them)
        float4 pv[2];
        float fcv[2];
        int mj = 0;                                            // metadata: threads pt < NR, row = pt
        float4 mu4 = make_float4(0.f, 0.f, 0.f, 0.f);
        auto load = [&](int k) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = rsub + 16 * h, g = r / EG;
                const int s = s_sb[g] + k * EG + (r % EG);
                const bool ok = s < s_se[g];
                const int sl = ok ? s : 0;
                const float fc = geo[(int64_t)sl * SPK_GEO_STRIDE + 4];
                fcv[h] = ok ? fc : 0.f;
                pv[h] = *reinterpret_cast<const float4*>(phi + (int64_t)sl * KP + (q_in ? qc * 4 : 0));
            }
            if (pt < NR) {
                const int g = pt / EG;
                const int s = s_sb[g] + k * EG + (pt % EG);
                const int sl = s < s_se[g] ? s : 0;
                mj = slot_j[sl];
                mu4 = *reinterpret_cast<const float4*>(geo + (int64_t)sl * SPK_GEO_STRIDE);   // ux uy uz d
            }
        };
        auto stage = [&](int k) {                              // Phi' = fc * [phi | 1]: the MMA yields W itself
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float4 v = with_bias(pv[h], q_in, qc, n_rbf);
                const float fc = fcv[h];
                v.x *= fc; v.y *= fc; v.z *= fc; v.w *= fc;
                put_row(sB, rsub + 16 * h, qc, v);
            }
            if (pt < NR) {
                uint8_t* m = sMeta + (k % NBUF) * META_F;
                reinterpret_cast<int*>(m)[pt] = mj;
                reinterpret_cast<float4*>(m + NR * 4)[pt] = mu4;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the stage is read by the async proxy
            wg_bar(PROD_BAR);
        };
        const uint32_t aB = smem_u32(sA), bB = smem_u32(sB);
        if (n_chunks > 0) {
            load(0);
            stage(0);
        }
        mbar_wait(&a_full, 0);
        for (int k = 0; k < n_chunks; ++k) {
            const int b = k % NBUF;
            const bool more = k + 1 < n_chunks;
            if (more) load(k + 1);                             // in flight during the MMAs of chunk k
            filter_to_tile<NT>(aB, bB, sT + b * T_FLOATS, pt);
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[b]);
            if (warp == W_PROD0 && k < 16) ETRACE(16 + k);
            if (more) {
                const int nb = (k + 1) % NBUF, use = (k + 1) / NBUF;
                if (use >= 1) mbar_wait(&empty_bar[nb], (use - 1) & 1);   // tile and metadata of chunk k+1-NBUF consumed
                wg_bar(PROD_BAR);                              // every warp's MMAs of chunk k have read the stage
                stage(k + 1);
            }
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
        for (int k = 0; k < n_chunks; ++k) {
            const int b = k % NBUF;
            if (warp == 0 && k < 16) ETRACE(64 + k);           // consumer 0: starts waiting
            mbar_wait(&full_bar[b], (k / NBUF) & 1);           // filter tile and metadata of the chunk
            if (warp == 0 && k < 16) ETRACE(176 + k);
            // this group's rows of the filter tile, thread = channel: read where they are used, which keeps 24 registers free
            const float* tg = sT + b * T_FLOATS + g * EG * T_LD + c;
            if (warp == 0 && k < 16) ETRACE(80 + k);           // filter values ready
            if (warp == 0 && lane == 0 && k == 0) SPK_TL_PHASE(2);
            const int* st_j = reinterpret_cast<const int*>(sMeta + b * META_F) + g * EG;
            const float4* st_u = reinterpret_cast<const float4*>(sMeta + b * META_F + NR * 4) + g * EG;
            const int base = s_begin + k * EG;
            // all eight gathers are issued before the first use (rows past the range read sender 0, their filter values
            // are exactly 0), so eight memory latencies overlap instead of following each other
            if (base < s_end) {
                float xa[EG], xb[EG], xc[EG], m0[EG], m1[EG], m2[EG];
#pragma unroll
                for (int u = 0; u < EG; ++u) {
#ifdef SPK_EDGE_EXP_JMASK
                    const int j = st_j[u] & 7;                 // experiment: all gathers hit L1 (timing only)
#else
                    const int j = st_j[u];
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
                for (int u = 0; u < EG; ++u) {
                    const int s = base + u;
                    if (s < s_end) {
                        while (s >= next_boundary) {
                            flush(i);
                            ++i;
                            next_boundary = boundary2;
                            prefetch_row(i);
                        }
                        const float4 uv = st_u[u];
                        dq = fmaf(tg[u * T_LD], xa[u], dq);
                        const float tb = tg[u * T_LD + F] * xb[u];
                        dm0 = fmaf(tb, uv.x, dm0);
                        dm1 = fmaf(tb, uv.y, dm1);
                        dm2 = fmaf(tb, uv.z, dm2);
                        if (HAS_MU) {
                            const float tc = tg[u * T_LD + 2 * F] * xc[u];
                            dm0 = fmaf(tc, m0[u], dm0);
                            dm1 = fmaf(tc, m1[u], dm1);
                            dm2 = fmaf(tc, m2[u], dm2);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[b]);
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
// A chunk is 4 groups x 4 edges.  Its operand has NR = 32 rows: rows 0..15 = fc [phi | 1] (-> W) and rows 16..31 =
// dfc [phi | 1] + fc [dphi | 0] (-> dW/dd), so one m64n32 product yields both the filter and its radial derivative.
constexpr int EGB = NR / 2 / NG;               // 4 edges per group and chunk
constexpr int NEB = EGB * NG;                  // 16 edges per chunk (x 2 operand rows each)
constexpr int META_B = NEB * 4 + NEB * 4 + NEB * 16;   // receiver index, edge id, (ux, uy, uz, 1/d) per edge
constexpr int SMEM_BYTES_B = A_BYTES + B_BYTES + NBUF * (T_BYTES + META_B) + 1024;


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
    float* sT = reinterpret_cast<float*>(sB + B_BYTES);
    uint8_t* sMeta = sB + B_BYTES + NBUF * T_BYTES;
    __shared__ __align__(8) uint64_t a_full, full_bar[NBUF], empty_bar[NBUF];
    __shared__ int s_rlo[NG], s_rhi[NG], s_sb[NG], s_se[NG];
    __shared__ float s_red[2][NG][EGB][4][4];      // [chunk parity][group][edge][warp][scalar]

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) {
        mbar_init(&a_full, 1);
#pragma unroll
        for (int b = 0; b < NBUF; ++b) {
            mbar_init(&full_bar[b], 4);
            mbar_init(&empty_bar[b], NCW);
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
        const int pt = tid - W_PROD0 * 32;
        const int qc = pt & 7, e = pt >> 3;                    // 8 x 16 B K-chunks per row, one edge per 8 threads
        const bool q_in = qc * 4 < KP;
        float4 pv, dv;
        float fc = 0.f, dfc = 0.f;
        int m_i = 0, m_e = 0;                                  // metadata: threads pt < NEB, edge = pt
        float4 m_u = make_float4(0.f, 0.f, 0.f, 0.f);
        auto load = [&](int k) {
            {
                const int g = e / EGB;
                const int pp = s_sb[g] + k * EGB + (e % EGB);
                const bool ok = pp < s_se[g];
                const int sl = pos_slot[ok ? pp : 0];
                const float2 f2 = *reinterpret_cast<const float2*>(geo + (int64_t)sl * SPK_GEO_STRIDE + 4);   // fc, dfc
                fc = ok ? f2.x : 0.f;
                dfc = ok ? f2.y : 0.f;
                pv = *reinterpret_cast<const float4*>(phi + (int64_t)sl * KP + (q_in ? qc * 4 : 0));
                dv = *reinterpret_cast<const float4*>(dphi + (int64_t)sl * KP + (q_in ? qc * 4 : 0));
            }
            if (pt < NEB) {
                const int g = pt / EGB;
                const int pp = s_sb[g] + k * EGB + (pt % EGB);
                const bool ok = pp < s_se[g];
                const int sl = pos_slot[ok ? pp : 0];
                m_i = pos_i[ok ? pp : 0];
                m_e = slot_eid[sl];
                const float4 g0 = *reinterpret_cast<const float4*>(geo + (int64_t)sl * SPK_GEO_STRIDE);
                m_u = make_float4(g0.x, g0.y, g0.z, geo[(int64_t)sl * SPK_GEO_STRIDE + 6]);
            }
        };
        auto stage = [&](int k) {                              // rows of the W and dW/dd operands
            const float4 v = with_bias(pv, q_in, qc, n_rbf);   // [phi | 1]
            float4 d = q_in ? dv : make_float4(0.f, 0.f, 0.f, 0.f);
            if (qc == (n_rbf >> 2)) {                          // bias column of [dphi | 0]
                const int kb = n_rbf & 3;
                if (kb == 0) d.x = 0.f; else if (kb == 1) d.y = 0.f; else if (kb == 2) d.z = 0.f; else d.w = 0.f;
            }
            float4 w, dw;
            w.x = fc * v.x; w.y = fc * v.y; w.z = fc * v.z; w.w = fc * v.w;
            dw.x = fmaf(dfc, v.x, fc * d.x); dw.y = fmaf(dfc, v.y, fc * d.y);
            dw.z = fmaf(dfc, v.z, fc * d.z); dw.w = fmaf(dfc, v.w, fc * d.w);
            put_row(sB, e, qc, w);
            put_row(sB, NEB + e, qc, dw);
            if (pt < NEB) {
                uint8_t* m = sMeta + (k % NBUF) * META_B;
                reinterpret_cast<int*>(m)[pt] = m_i;
                reinterpret_cast<int*>(m)[NEB + pt] = m_e;
                reinterpret_cast<float4*>(m + 2 * NEB * 4)[pt] = m_u;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            wg_bar(PROD_BAR);
        };
        const uint32_t aB = smem_u32(sA), bB = smem_u32(sB);
        if (n_chunks > 0) {
            load(0);
            stage(0);
        }
        mbar_wait(&a_full, 0);
        for (int k = 0; k < n_chunks; ++k) {
            const int b = k % NBUF;
            const bool more = k + 1 < n_chunks;
            if (more) load(k + 1);
            filter_to_tile<NT>(aB, bB, sT + b * T_FLOATS, pt);
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[b]);
            if (warp == W_PROD0 && k < 16) BTRACE(16 + k);
            if (more) {
                const int nb = (k + 1) % NBUF, use = (k + 1) / NBUF;
                if (use >= 1) mbar_wait(&empty_bar[nb], (use - 1) & 1);
                wg_bar(PROD_BAR);
                stage(k + 1);
            }
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
        for (int k = 0; k < n_chunks; ++k) {
            const int b = k % NBUF;
            if (warp == 0 && k < 16) BTRACE(64 + k);           // consumer 0: starts waiting
            mbar_wait(&full_bar[b], (k / NBUF) & 1);           // filter tile and metadata of the chunk
            if (warp == 0 && k < 16) BTRACE(176 + k);
            const float* tg = sT + b * T_FLOATS + g * EGB * T_LD + c;   // W rows of the group; dW/dd rows NEB further
            float Wv[3][EGB], Dv[3][EGB];
#pragma unroll
            for (int t = 0; t < NT; ++t)
#pragma unroll
                for (int u = 0; u < EGB; ++u) {
                    Wv[t][u] = tg[u * T_LD + t * F];
                    Dv[t][u] = tg[(NEB + u) * T_LD + t * F];
                }
            if (warp == 0 && k < 16) BTRACE(80 + k);           // filter values ready
            if (warp == 0 && lane == 0 && k == 0) SPK_TL_PHASE(2);
            const int* st_i = reinterpret_cast<const int*>(sMeta + b * META_B) + g * EGB;
            const int* st_e = reinterpret_cast<const int*>(sMeta + b * META_B) + NEB + g * EGB;
            const float4* st_u = reinterpret_cast<const float4*>(sMeta + b * META_B + 2 * NEB * 4) + g * EGB;
            const int base = p_begin + k * EGB;
            {
                float gq[EGB], g0[EGB], g1[EGB], g2[EGB];
#pragma unroll
                for (int u = 0; u < EGB; ++u) {                // rows past the range gather receiver 0; their W, dW are 0
                    const int i = st_i[u];
                    gq[u] = g_q[(size_t)i * F + c];
                    const float* __restrict__ gmi = g_mu + (size_t)i * (3 * F) + c;
                    g0[u] = gmi[0];
                    g1[u] = gmi[F];
                    g2[u] = gmi[2 * F];
                }
                float red[16];
#pragma unroll
                for (int u = 0; u < EGB; ++u) {
                    const int p = base + u;
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
                        const float4 ge = st_u[u];                 // ux uy uz 1/d
                        const float gu = g0[u] * ge.x + g1[u] * ge.y + g2[u] * ge.z;
                        gxa = fmaf(Wv[0][u], gq[u], gxa);
                        gxb = fmaf(Wv[1][u], gu, gxb);
                        part_d = gq[u] * xa * Dv[0][u] + gu * xb * Dv[1][u];
                        const float wbx = Wv[1][u] * xb;
                        pu0 = g0[u] * wbx;
                        pu1 = g1[u] * wbx;
                        pu2 = g2[u] * wbx;
                        if (HAS_MU) {
                            const float gm = g0[u] * m0 + g1[u] * m1 + g2[u] * m2;
                            gxc = fmaf(Wv[2][u], gm, gxc);
                            const float wcx = Wv[2][u] * xc;
                            gm0 = fmaf(wcx, g0[u], gm0);
                            gm1 = fmaf(wcx, g1[u], gm1);
                            gm2 = fmaf(wcx, g2[u], gm2);
                            part_d = fmaf(gm * xc, Dv[2][u], part_d);
                        }
                    }
                    red[4 * u + 0] = part_d;
                    red[4 * u + 1] = pu0;
                    red[4 * u + 2] = pu1;
                    red[4 * u + 3] = pu2;
                }
                const float tot = butterfly16(red, lane);
                if (!(lane & 1)) s_red[k & 1][g][my_idx >> 2][qd][my_idx & 3] = tot;
            }
            // the four warps of the group have published their partial sums of this chunk's edges
            asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
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
            if (lane == 0) mbar_arrive(&empty_bar[b]);
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
    if (nb > spk_cdiv(n_edges, NR)) nb = spk_cdiv(n_edges, NR);
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

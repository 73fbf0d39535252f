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
//   * one persistent CTA per SM: 4 consumer warpgroups forward (a group owns 128 channels of its own edge-balanced
//     receiver range, as a CTA of painn.cu did), 8 consumer warps reverse (a warp owns its own edge-balanced sender range,
//     a lane 4 channels), and one producer warpgroup.  The producer stages the Phi' rows of a whole chunk (every
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
// Reverse: 64+k the chunk starts, 80+k the gathers of chunk k+1 are issued and the wait starts, 176+k it returns, 96+k
// the chunk is done (its g_rij included).

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
constexpr int K_TC = 24;                       // K = n_rbf + 1 covered by the three k-steps of filter_third
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
// reverse pass, grouped by sender (reference: autograd of painn.py:55-65)
// ------------------------------------------------------------------------------------------------------------------
// One persistent CTA per SM of 8 consumer warps and the producer warpgroup (384 threads, up to 168 registers each).  Each
// consumer WARP owns an edge-balanced sender range and 2 edges of every chunk; a lane owns 4 channels and reads them as
// float4.  A chunk is 8 warps x 2 edges; its operand has NR = 32 rows: rows 0..15 = fc [phi | 1] (-> W) and rows 16..31 =
// dfc [phi | 1] + fc [dphi | 0] (-> dW/dd), so one m64n32 product yields both the filter and its radial derivative.
// A warp finds the receivers of its own edges (pos_i over its contiguous range), so the g_q / g_mu gathers of chunk k+1
// are in flight before it waits for the filter tile of chunk k.  The four per-edge channel sums (dE/dd, dE/du) end
// inside the warp, and the warp writes its edges' g_rij: no barrier between the consumer warps.
constexpr int NCW_B = 8;                       // consumer warps
constexpr int W_PROD0_B = NCW_B;               // the producer warpgroup: warps NCW_B .. NCW_B + 3
constexpr int NTHREADS_B = (NCW_B + 4) * 32;
constexpr int PROD_BAR_B = 1;                  // named barrier of the producer warpgroup
constexpr int EGB = NR / 2 / NCW_B;            // 2 edges per warp and chunk
constexpr int NEB = EGB * NCW_B;               // 16 edges per chunk (x 2 operand rows each)
constexpr int WIN = 32 / EGB;                  // chunks per index window (one edge per lane)
constexpr int META_B = NEB * 16;               // (ux, uy, uz, 1/d) per edge
constexpr int SMEM_BYTES_B = A_BYTES + B_BYTES + NBUF * (T_BYTES + META_B) + 1024;

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// Sum over the 32 lanes of 8 values per lane (2 edges x 4 scalars) with a transposing butterfly: 9 shuffles.  Afterwards
// lane l holds the complete sum of value index 4*bit4 + 2*bit3 + bit2 (all four lanes of a quad).
__device__ __forceinline__ float butterfly8(float (&v)[8], int lane) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const bool up = lane & 16;
        const float send = up ? v[i] : v[i + 4];
        const float keep = up ? v[i + 4] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const bool up = lane & 8;
        const float send = up ? v[i] : v[i + 2];
        const float keep = up ? v[i + 2] : v[i];
        v[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    {
        const bool up = lane & 4;
        const float send = up ? v[0] : v[1];
        const float keep = up ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
    return v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
}

// One channel of one edge: the sender accumulators (the expressions of the one-thread-per-channel kernel, so g_x and
// g_mu_in do not depend on how channels map to lanes) and this channel's share of the four per-edge scalars in s.
template <bool HAS_MU>
__device__ __forceinline__ void bwd_channel(float gq, float g0, float g1, float g2, float4 ge, float w0, float w1,
                                            float w2, float d0, float d1, float d2, float xa, float xb, float xc,
                                            float m0, float m1, float m2, float& gxa, float& gxb, float& gxc,
                                            float& gm0, float& gm1, float& gm2, float (&s)[4]) {
    const float gu = g0 * ge.x + g1 * ge.y + g2 * ge.z;
    gxa = fmaf(w0, gq, gxa);
    gxb = fmaf(w1, gu, gxb);
    float part_d = gq * xa * d0 + gu * xb * d1;
    const float wbx = w1 * xb;
    if (HAS_MU) {
        const float gm = g0 * m0 + g1 * m1 + g2 * m2;
        gxc = fmaf(w2, gm, gxc);
        const float wcx = w2 * xc;
        gm0 = fmaf(wcx, g0, gm0);
        gm1 = fmaf(wcx, g1, gm1);
        gm2 = fmaf(wcx, g2, gm2);
        part_d = fmaf(gm * xc, d2, part_d);
    }
    s[0] += part_d;
    s[1] += g0 * wbx;
    s[2] += g1 * wbx;
    s[3] += g2 * wbx;
}

template <bool HAS_MU>
__global__ void __launch_bounds__(NTHREADS_B, 1) k_painn_edge_bwd_tc(
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
    __shared__ int s_rlo[NCW_B], s_rhi[NCW_B], s_sb[NCW_B], s_se[NCW_B];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) {
        mbar_init(&a_full, 1);
#pragma unroll
        for (int b = 0; b < NBUF; ++b) {
            mbar_init(&full_bar[b], 4);
            mbar_init(&empty_bar[b], NCW_B);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(&a_full, A_BYTES);          // static operand: fetched BEFORE griddepcontrol.wait (pack kernels never trigger their dependents early, common.cuh)
        tma_load(sA, wpk, A_BYTES, &a_full);
    }
    if (tid == 0) BTRACE(0);
    SPK_PDL_WAIT();
    if (tid == 0) BTRACE(1);
    if (warp <= NCW_B) {                           // warp w finds boundary w of this CTA's NCW_B warp ranges (warp-wide search)
        const int bnd = spk_block_row_begin_warp(sptr, n_atoms, n_edges, gridDim.x * NCW_B, blockIdx.x * NCW_B + warp);
        if (lane == 0) {
            const int e = sptr[bnd];
            if (warp < NCW_B) {
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
    for (int w = 0; w < NCW_B; ++w) n_chunks = max(n_chunks, (s_se[w] - s_sb[w] + EGB - 1) / EGB);
    const int KP = spk_kp(n_rbf);

    if (warp >= W_PROD0_B) {
        // =========================================== producers ===========================================
        const int pt = tid - W_PROD0_B * 32;
        const int qc = pt & 7, e = pt >> 3;                    // 8 x 16 B K-chunks per row, one edge per 8 threads
        const bool q_in = qc * 4 < KP;
        // Edge ed of chunk k: its position in the sender grouping (0 past the warp's range), ok = inside the range.
        auto edge_pos = [&](int k, int ed, bool& ok) {
            const int w = ed / EGB;
            const int pp = s_sb[w] + k * EGB + (ed % EGB);
            ok = pp < s_se[w];
            return ok ? pp : 0;
        };
        // The global loads run two chunks ahead of the MMAs, in two register sets that alternate with the chunk's parity:
        // set k % 2 holds the rows of chunk k until they are staged, then those of chunk k+2, and the slots of chunk
        // k+2, then those of chunk k+4.  A load then has two chunk periods to land, and no load waits for its slot.
        struct Rows {
            float4 pv, dv;                                     // phi, dphi of the row edge (16 B K-chunk qc)
            float2 fcd;                                        // fc, dfc of the row edge
            float4 m_u;                                        // metadata: threads pt < NEB, edge = pt
            bool ok;                                           // the row edge lies inside its warp's range
            int sl, sl_m;                                      // slots of the chunk loaded next into this set
        };
        auto load_slots = [&](Rows& r, int k) {
            bool ok;
            r.sl = pos_slot[edge_pos(k, e, ok)];
            if (pt < NEB) r.sl_m = pos_slot[edge_pos(k, pt, ok)];
        };
        // Nothing here reads the loaded values; stage() is the first (masking fc, dfc of rows past a range included).
        auto load = [&](Rows& r, int k) {                      // the slots of chunk k are in r.sl, r.sl_m
            edge_pos(k, e, r.ok);
            r.fcd = *reinterpret_cast<const float2*>(geo + (int64_t)r.sl * SPK_GEO_STRIDE + 4);
            r.pv = *reinterpret_cast<const float4*>(phi + (int64_t)r.sl * KP + (q_in ? qc * 4 : 0));
            r.dv = *reinterpret_cast<const float4*>(dphi + (int64_t)r.sl * KP + (q_in ? qc * 4 : 0));
            if (pt < NEB) {
                const float4 g0 = *reinterpret_cast<const float4*>(geo + (int64_t)r.sl_m * SPK_GEO_STRIDE);
                r.m_u = make_float4(g0.x, g0.y, g0.z, geo[(int64_t)r.sl_m * SPK_GEO_STRIDE + 6]);
            }
        };
        auto stage = [&](const Rows& r, int k) {               // rows of the W and dW/dd operands
            const float fc = r.ok ? r.fcd.x : 0.f, dfc = r.ok ? r.fcd.y : 0.f;
            const float4 v = with_bias(r.pv, q_in, qc, n_rbf); // [phi | 1]
            float4 d = q_in ? r.dv : make_float4(0.f, 0.f, 0.f, 0.f);
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
            if (pt < NEB) reinterpret_cast<float4*>(sMeta + (k % NBUF) * META_B)[pt] = r.m_u;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            wg_bar(PROD_BAR_B);
        };
        const uint32_t aB = smem_u32(sA), bB = smem_u32(sB);
        Rows ra{}, rb{};
        if (n_chunks > 0) {
            load_slots(ra, 0);
            if (n_chunks > 1) load_slots(rb, 1);
            load(ra, 0);
            if (n_chunks > 1) load(rb, 1);
            if (n_chunks > 2) load_slots(ra, 2);
            if (n_chunks > 3) load_slots(rb, 3);
            stage(ra, 0);
        }
        mbar_wait(&a_full, 0);
        auto step = [&](int k, Rows& cur, Rows& nxt) {         // cur: chunk k, staged; nxt: chunk k+1
            const int b = k % NBUF;
            if (k + 2 < n_chunks) {
                load(cur, k + 2);
                if (k + 4 < n_chunks) load_slots(cur, k + 4);
            }
            filter_to_tile<NT>(aB, bB, sT + b * T_FLOATS, pt);
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[b]);
            if (warp == W_PROD0_B && k < 16) BTRACE(16 + k);
            if (k + 1 < n_chunks) {
                const int nb = (k + 1) % NBUF, use = (k + 1) / NBUF;
                if (use >= 1) mbar_wait(&empty_bar[nb], (use - 1) & 1);
                wg_bar(PROD_BAR_B);
                stage(nxt, k + 1);
            }
        };
        for (int k = 0; k < n_chunks; k += 2) {                // the two register sets stay in fixed registers
            step(k, ra, rb);
            if (k + 1 < n_chunks) step(k + 1, rb, ra);
        }
    } else {
        // =========================================== consumers ===========================================
        const int c = lane * 4;                                // this lane's four channels
        const int j_hi = s_rhi[warp], p_begin = s_sb[warp], p_end = s_se[warp];
        const int n_mine = (p_end - p_begin + EGB - 1) / EGB;  // chunks with edges of this warp
        const int n_win = (p_end - p_begin + 31) / 32;
        int j = s_rlo[warp];
        int next_boundary = j < j_hi ? sptr[j + 1] : 0x7fffffff;
        int boundary2 = j + 1 < j_hi ? sptr[j + 2] : 0x7fffffff;
        const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 xa = z4, xb = z4, xc = z4, m0 = z4, m1 = z4, m2 = z4;
        float4 gxa = z4, gxb = z4, gxc = z4, gm0 = z4, gm1 = z4, gm2 = z4;
        auto load_own = [&](int row) {
            const float* __restrict__ xr = x + (size_t)row * (3 * F) + c;
            xa = ld4(xr);
            xb = ld4(xr + F);
            if (HAS_MU) {
                xc = ld4(xr + 2 * F);
                const float* __restrict__ mr = mu + (size_t)row * (3 * F) + c;
                m0 = ld4(mr);
                m1 = ld4(mr + F);
                m2 = ld4(mr + 2 * F);
            }
        };
        auto flush = [&](int row) {
            const size_t o = (size_t)row * 3 * F + c;
            float4 r0, r1, r2;
            if (HAS_MU) {                                      // residual: issued before the stores
                r0 = ld4(g_mu + o);
                r1 = ld4(g_mu + o + F);
                r2 = ld4(g_mu + o + 2 * F);
            }
            st4(g_x + o, gxa);
            st4(g_x + o + F, gxb);
            st4(g_x + o + 2 * F, gxc);
            if (HAS_MU) {
                st4(g_mu_in + o, make_float4(r0.x + gm0.x, r0.y + gm0.y, r0.z + gm0.z, r0.w + gm0.w));
                st4(g_mu_in + o + F, make_float4(r1.x + gm1.x, r1.y + gm1.y, r1.z + gm1.z, r1.w + gm1.w));
                st4(g_mu_in + o + 2 * F, make_float4(r2.x + gm2.x, r2.y + gm2.y, r2.z + gm2.z, r2.w + gm2.w));
            }
            gxa = gxb = gxc = gm0 = gm1 = gm2 = z4;
        };
        // Edge p is past the current row: flush it and any edge-free rows after it, and move to the row of p.  The own
        // rows of the new sender are loaded before the flush, so their latency and that of the residual overlap.
        auto next_row = [&](int p) {
            int j2 = j + 1, nbd = boundary2;
            while (p >= nbd) nbd = sptr[++j2 + 1];
            load_own(j2);
            flush(j);
            for (int r = j + 1; r < j2; ++r) flush(r);
            j = j2;
            next_boundary = nbd;
            boundary2 = j + 1 < j_hi ? sptr[j + 2] : 0x7fffffff;
        };
        if (j < j_hi) load_own(j);

        // Index windows: lane l holds receiver, edge id and (accumulate) the old g_rij of edge p_begin + 32 w + l, the
        // edges of chunks WIN w .. WIN w + WIN-1.  The next window is filled in three steps spread over the current
        // one (pos_i + pos_slot, slot_eid, g_rij), so no chunk waits on that chain.
        int wi = 0, we = 0, ni = 0, ne = 0;
        float wr0 = 0.f, wr1 = 0.f, wr2 = 0.f, nr0 = 0.f, nr1 = 0.f, nr2 = 0.f;
        auto win_idx = [&](int w, int& i_, int& e_) {          // e_: the slot until win_eid
            const int p = p_begin + 32 * w + lane;
            if (p < p_end) {
                i_ = pos_i[p];
                e_ = pos_slot[p];
            }
        };
        auto win_eid = [&](int w, int& e_) {
            if (p_begin + 32 * w + lane < p_end) e_ = slot_eid[e_];
        };
        auto win_old = [&](int w, int e_, float& a, float& b_, float& c_) {
            if (accumulate && p_begin + 32 * w + lane < p_end) {
                const float* o = g_rij + (int64_t)e_ * 3;
                a = o[0];
                b_ = o[1];
                c_ = o[2];
            }
        };
        // g_q and g_mu rows of the receivers of chunk q's edges, [edge][g_q, g_mu x, y, z]
        auto gather = [&](float4 (&G)[EGB][4], int q, int src_i) {
#pragma unroll
            for (int u = 0; u < EGB; ++u) {
                const int i = __shfl_sync(0xffffffffu, src_i, (q * EGB + u) & 31);
                if (p_begin + q * EGB + u < p_end) {
                    G[u][0] = ld4(g_q + (size_t)i * F + c);
                    const float* __restrict__ gmi = g_mu + (size_t)i * (3 * F) + c;
                    G[u][1] = ld4(gmi);
                    G[u][2] = ld4(gmi + F);
                    G[u][3] = ld4(gmi + 2 * F);
                }
            }
        };
        float4 ga[EGB][4], gb[EGB][4];
        if (n_mine > 0) {
            win_idx(0, wi, we);
            if (n_win > 1) win_idx(1, ni, ne);
            gather(ga, 0, wi);
            win_eid(0, we);
            win_old(0, we, wr0, wr1, wr2);
        }

        auto step = [&](int k, float4 (&G)[EGB][4], float4 (&Gn)[EGB][4]) {
            const int b = k % NBUF;
            if (warp == 0 && k < 16) BTRACE(64 + k);           // consumer 0: the chunk starts
            if (k + 1 < n_mine) gather(Gn, k + 1, (k + 1) % WIN == 0 ? ni : wi);
            if (warp == 0 && k < 16) BTRACE(80 + k);           // gathers of the next chunk issued, starts waiting
            mbar_wait(&full_bar[b], (k / NBUF) & 1);           // filter tile and metadata of the chunk
            if (warp == 0 && k < 16) BTRACE(176 + k);
            if (warp == 0 && lane == 0 && k == 0) SPK_TL_PHASE(2);
            const float4* st_u = reinterpret_cast<const float4*>(sMeta + b * META_B) + warp * EGB;
            if (k < n_mine) {
                // this warp's rows of the filter tile, read where they are used; dW/dd rows NEB further
                const float* tw = sT + b * T_FLOATS + warp * EGB * T_LD + c;
                const int base = p_begin + k * EGB;
                float red[4 * EGB];
#pragma unroll
                for (int u = 0; u < EGB; ++u) {
                    float s[4] = {0.f, 0.f, 0.f, 0.f};
                    if (base + u < p_end) {
                        if (base + u >= next_boundary) next_row(base + u);
                        const float4 ge = st_u[u];             // ux uy uz 1/d
                        const float4 w0 = ld4(tw + u * T_LD), w1 = ld4(tw + u * T_LD + F);
                        const float4 d0 = ld4(tw + (NEB + u) * T_LD), d1 = ld4(tw + (NEB + u) * T_LD + F);
                        const float4 w2 = HAS_MU ? ld4(tw + u * T_LD + 2 * F) : z4;
                        const float4 d2 = HAS_MU ? ld4(tw + (NEB + u) * T_LD + 2 * F) : z4;
                        const float4 gq = G[u][0], g0 = G[u][1], g1 = G[u][2], g2 = G[u][3];
                        bwd_channel<HAS_MU>(gq.x, g0.x, g1.x, g2.x, ge, w0.x, w1.x, w2.x, d0.x, d1.x, d2.x, xa.x, xb.x,
                                            xc.x, m0.x, m1.x, m2.x, gxa.x, gxb.x, gxc.x, gm0.x, gm1.x, gm2.x, s);
                        bwd_channel<HAS_MU>(gq.y, g0.y, g1.y, g2.y, ge, w0.y, w1.y, w2.y, d0.y, d1.y, d2.y, xa.y, xb.y,
                                            xc.y, m0.y, m1.y, m2.y, gxa.y, gxb.y, gxc.y, gm0.y, gm1.y, gm2.y, s);
                        bwd_channel<HAS_MU>(gq.z, g0.z, g1.z, g2.z, ge, w0.z, w1.z, w2.z, d0.z, d1.z, d2.z, xa.z, xb.z,
                                            xc.z, m0.z, m1.z, m2.z, gxa.z, gxb.z, gxc.z, gm0.z, gm1.z, gm2.z, s);
                        bwd_channel<HAS_MU>(gq.w, g0.w, g1.w, g2.w, ge, w0.w, w1.w, w2.w, d0.w, d1.w, d2.w, xa.w, xb.w,
                                            xc.w, m0.w, m1.w, m2.w, gxa.w, gxb.w, gxc.w, gm0.w, gm1.w, gm2.w, s);
                    }
#pragma unroll
                    for (int t = 0; t < 4; ++t) red[4 * u + t] = s[t];
                }
                // lane 16 u + 4 t holds scalar t (dE/dd, dE/du x, y, z) of edge u; lane 16 u writes the edge's g_rij
                const float v = butterfly8(red, lane);
                const float u0 = __shfl_down_sync(0xffffffffu, v, 4);
                const float u1 = __shfl_down_sync(0xffffffffu, v, 8);
                const float u2 = __shfl_down_sync(0xffffffffu, v, 12);
                const int src = (k * EGB + (lane >> 4)) & 31;  // the edge's lane in the index window
                const int eid = __shfl_sync(0xffffffffu, we, src);
                const float o0 = __shfl_sync(0xffffffffu, wr0, src);
                const float o1 = __shfl_sync(0xffffffffu, wr1, src);
                const float o2 = __shfl_sync(0xffffffffu, wr2, src);
                if ((lane & 15) == 0 && base + (lane >> 4) < p_end) {
                    const float4 ge = st_u[lane >> 4];
                    const float dot = u0 * ge.x + u1 * ge.y + u2 * ge.z;
                    float r0 = v * ge.x + (u0 - dot * ge.x) * ge.w;
                    float r1 = v * ge.y + (u1 - dot * ge.y) * ge.w;
                    float r2 = v * ge.z + (u2 - dot * ge.z) * ge.w;
                    if (accumulate) {
                        r0 += o0;
                        r1 += o1;
                        r2 += o2;
                    }
                    float* out = g_rij + (int64_t)eid * 3;
                    out[0] = r0;
                    out[1] = r1;
                    out[2] = r2;
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[b]);
            if (warp == 0 && k < 16) BTRACE(96 + k);           // chunk done (incl. its g_rij)
            // the next window's steps; at the window's end it becomes the current one
            const int kw = k / WIN, kk = k % WIN;
            if (kw + 1 < n_win) {
                if (kk == 4) win_eid(kw + 1, ne);
                if (kk == 8) win_old(kw + 1, ne, nr0, nr1, nr2);
                if (kk == WIN - 1) {
                    wi = ni;
                    we = ne;
                    wr0 = nr0;
                    wr1 = nr1;
                    wr2 = nr2;
                    if (kw + 2 < n_win) win_idx(kw + 2, ni, ne);
                }
            }
        };
        for (int k = 0; k < n_chunks; k += 2) {                // two gather buffers in fixed registers
            step(k, ga, gb);
            if (k + 1 < n_chunks) step(k + 1, gb, ga);
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
    if (F != F_TC || n_rbf <= 0 || n_rbf + 1 > K_TC) return SPK_ERR_UNSUPPORTED;
    spk_launch(k_pack_filter, (unsigned)spk_cdiv(3 * F_TC * 32, 256), 256, 0, spk_st(stream), wf, bf, n_rbf, packed);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_painn_edge_fwd_tc(const float* x, const float* mu, const float* q, const float* phi, const float* geo,
                                     const int32_t* rowptr, const int32_t* slot_j, const float* wf_packed,
                                     int64_t n_atoms, int64_t n_edges, int F, int n_rbf, float* q_out, float* mu_out,
                                     spk_stream_t stream) {
    if (n_atoms < 0 || n_edges < 0 || F <= 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (F != F_TC || n_rbf + 1 > K_TC || n_edges == 0) return SPK_ERR_UNSUPPORTED;      // caller uses spk_painn_edge_fwd
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
    if (F != F_TC || n_rbf + 1 > K_TC || n_edges == 0) return SPK_ERR_UNSUPPORTED;      // caller uses spk_painn_edge_bwd
    if (n_atoms == 0) return SPK_OK;
    if (!x || !g_q || !g_mu || !phi || !dphi || !geo || !sptr || !pos_slot || !pos_i || !slot_eid || !wf_packed || !g_x ||
        !g_rij)
        return SPK_ERR_ARG;
    if (mu && !g_mu_in) return SPK_ERR_ARG;
    if ((reinterpret_cast<uintptr_t>(phi) | reinterpret_cast<uintptr_t>(dphi) | reinterpret_cast<uintptr_t>(geo) |
         reinterpret_cast<uintptr_t>(wf_packed) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(mu) |
         reinterpret_cast<uintptr_t>(g_q) | reinterpret_cast<uintptr_t>(g_mu) | reinterpret_cast<uintptr_t>(g_x) |
         reinterpret_cast<uintptr_t>(g_mu_in)) & 15)                               // float4 rows
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
        spk_launch(k_painn_edge_bwd_tc<true>, (unsigned)nb, NTHREADS_B, SMEM_BYTES_B, st, x, mu, g_q, g_mu, phi, dphi, geo, sptr,
                   pos_slot, pos_i, slot_eid, wf_packed, (int)n_atoms, (int)n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate);
    else
        spk_launch(k_painn_edge_bwd_tc<false>, (unsigned)nb, NTHREADS_B, SMEM_BYTES_B, st, x, mu, g_q, g_mu, phi, dphi, geo, sptr,
                   pos_slot, pos_i, slot_eid, wf_packed, (int)n_atoms, (int)n_edges, n_rbf, g_x, g_mu_in, g_rij, accumulate);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

// Persistent per-atom stage ("atom chain"): ALL the per-atom work that sits between two fused edge kernels of a PaiNN
// evaluation -- mu_channel_mix, norm/context glue, intraatomic_context_net (2 Dense), gated update, and the NEXT block's
// interatomic_context_net (2 Dense); or their reverses -- as ONE launch (reference: representation/painn.py and
// nn/base.py; otherwise 7 launches per stage, each paying barrier set-up, pipeline fill and a full grid drain).
//
// Every operation of the stage is ROW-LOCAL: the rows of a 128-atom tile produced by step k are all that step k+1 needs
// for the same tile.  So the stage is a static list of STEPS (GEMM or elementwise glue, given by the host as plain structs)
// cut into WORK ITEMS (step, atom tile, sub-tile).  Items are numbered step-major and CLAIMED in increasing order from a
// global counter by one persistent CTA per SM; item (k, r, *) may start when the counter done[k-1][r] has reached the number
// of items of step k-1 for tile r (spin on ld.acquire, published with __threadfence + atomicAdd after the item's
// epilogue).  An item only waits for lower-numbered ones, and those are held by CTAs that are already running, so the
// schedule cannot deadlock however many CTAs are co-resident.  Data between steps goes through global memory (L2-resident,
// read with ld.global.cg): what is saved is the launch boundary, not the bytes.
//
// A GEMM item is one 128 x 128 output tile computed by the warp-specialised wgmma pipeline of gemm_tc.cu (3xTF32 with a
// fresh accumulator per K-tile added to fp32 registers, see there), kept WARM across items: the mbarrier phases run on
// (stage = global K-tile count % NST), weight tiles still arrive pre-packed by one TMA bulk copy each.  Activation codes and
// the "x act'(pre)" prologue are run-time here (one kernel, any program).
//
// The last CTA to finish resets the dependency counters, so the caller-owned workspace only has to be zero once.
#include "wgmma.cuh"

namespace {

constexpr int TM = 128, TN = 128, TK = 16;
constexpr int N_CONS = 8, W_PROD0 = 8;
constexpr int NST = 6, NPROD = 6;
constexpr int OPER_A = TM * TK * 4, OPER_B = TN * TK * 4;
constexpr int STAGE_BYTES = 2 * OPER_A + 2 * OPER_B;        // A_hi, A_lo, W_hi, W_lo
constexpr int EP_LD = TN + 4;
constexpr int SMEM_BYTES = NST * STAGE_BYTES + 1024;
constexpr int NTHREADS = (W_PROD0 + NPROD) * 32;            // 448
constexpr int NB = TN / 64;                                 // m64n64 column blocks per consumer warpgroup
static_assert(NST * STAGE_BYTES >= TM * EP_LD * 4, "epilogue staging tile reuses the pipeline stages");
static_assert(NST % NPROD == 0, "a stage must be owned by exactly one producer warp");

struct ChainArgs {
    spk_chain_step_t step[SPK_CHAIN_MAX_STEPS];
    int n_steps;
    int n_tiles;            // ceil(n_atoms / 128)
    int64_t n_atoms;
    int* ws;                // [n_steps * n_tiles] done counters, then [1] finished-CTA counter, [1] next-item counter
    long long* trace;       // optional (spk_atom_chain_debug): 8 stamps per item
};

__device__ __forceinline__ long long gtime() {
    long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
#define CTRACE(slot, val)                                                        \
    do {                                                                         \
        if (g.trace && tid == 0) g.trace[(int64_t)item * 8 + (slot)] = (val);    \
    } while (0)

__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ float4 ldcg4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ int items_per_tile(const spk_chain_step_t& s) {
    return s.kind == SPK_CHAIN_GEMM ? s.rows_per_atom * (s.N / TN) : 1;
}

// activation value and derivative for the epilogue of a 128 x 128 tile: 16 k elements on ONE SM, so the instruction count per
// element is what the tile's latency pays (expf + two IEEE divisions per element).  silu keeps expf
// (accuracy of the reference's sigmoid) but takes ONE reciprocal; shifted softplus as in common.cuh.
__device__ __forceinline__ void chain_act_both(float x, int act, float& y, float& dy) {
    if (act == SPK_ACT_SILU) {
        const float s = __frcp_rn(1.0f + expf(-x));
        y = x * s;
        dy = s * fmaf(x, 1.0f - s, 1.0f);
    } else {
        spk_act_both(x, act, y, dy);
    }
}

// ---- elementwise glue over the atoms [a0, a1) of one tile: 4 channels per thread, all threads of the CTA ------------------
__device__ __forceinline__ float4 f4_fma(float4 a, float4 b, float4 c) {
    return make_float4(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y), fmaf(a.z, b.z, c.z), fmaf(a.w, b.w, c.w));
}
__device__ __forceinline__ float4 f4_mul(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// element t of a tile -> (atom, channel group) with 32-bit arithmetic only
#define GLUE_LOOP_BEGIN                                                   \
    for (int t = tid; t < n; t += NTHREADS) {                             \
        const int ar = t / F4;                                            \
        const int64_t a = a0 + ar;                                        \
        const int c = (t - ar * F4) * 4;

__device__ void glue_item(const spk_chain_step_t& s, int64_t a0, int64_t a1, int tid) {
    const int F = s.F, F4 = F >> 2;
    const int n = (int)(a1 - a0) * F4;
    if (s.kind == SPK_CHAIN_MIX_CTX) {              // painn.py:104-107   g0 = q, g1 = VW -> o0 = ctx [N,2F]
#pragma unroll 2
        GLUE_LOOP_BEGIN
            const float* v = s.g1 + a * 6 * F + c;
            const float4 v0 = ldcg4(v), v1 = ldcg4(v + 2 * F), v2 = ldcg4(v + 4 * F);
            const float4 q = ldcg4(s.g0 + a * F + c);
            float4 nn = f4_fma(v2, v2, f4_fma(v1, v1, f4_mul(v0, v0)));
            nn = make_float4(sqrtf(nn.x + s.eps), sqrtf(nn.y + s.eps), sqrtf(nn.z + s.eps), sqrtf(nn.w + s.eps));
            st4(s.o0 + a * 2 * F + c, q);
            st4(s.o0 + a * 2 * F + F + c, nn);
        }
    } else if (s.kind == SPK_CHAIN_MIX_UPDATE) {    // painn.py:110-116   g0 = q, g1 = VW, g2 = mu, g3 = s -> o0 = q', o1 = mu'
#pragma unroll 1
        GLUE_LOOP_BEGIN
            const float* vw = s.g1 + a * 6 * F + c;
            const float4 v0 = ldcg4(vw), w0 = ldcg4(vw + F), v1 = ldcg4(vw + 2 * F), w1 = ldcg4(vw + 3 * F),
                         v2 = ldcg4(vw + 4 * F), w2 = ldcg4(vw + 5 * F);
            const float* sr = s.g3 + a * 3 * F + c;
            const float4 s1 = ldcg4(sr), s2 = ldcg4(sr + F), s3 = ldcg4(sr + 2 * F);
            const float4 q = ldcg4(s.g0 + a * F + c);
            const float* mr = s.g2 + a * 3 * F + c;
            const float4 m0 = ldcg4(mr), m1 = ldcg4(mr + F), m2 = ldcg4(mr + 2 * F);
            const float4 svw = f4_fma(v2, w2, f4_fma(v1, w1, f4_mul(v0, w0)));
            st4(s.o0 + a * F + c, f4_add(f4_add(q, s1), f4_mul(s3, svw)));
            float* mo = s.o1 + a * 3 * F + c;
            st4(mo, f4_fma(s2, w0, m0));
            st4(mo + F, f4_fma(s2, w1, m1));
            st4(mo + 2 * F, f4_fma(s2, w2, m2));
        }
    } else if (s.kind == SPK_CHAIN_MIX_UPDATE_BWD) { // g0 = g_q, g1 = VW, g2 = g_mu, g3 = s -> o0 = g_s [N,3F], o1 = g_VW [N,3,2F]
#pragma unroll 1
        GLUE_LOOP_BEGIN
            const float* vw = s.g1 + a * 6 * F + c;
            const float4 v0 = ldcg4(vw), w0 = ldcg4(vw + F), v1 = ldcg4(vw + 2 * F), w1 = ldcg4(vw + 3 * F),
                         v2 = ldcg4(vw + 4 * F), w2 = ldcg4(vw + 5 * F);
            const float* sr = s.g3 + a * 3 * F + c;
            const float4 s2 = ldcg4(sr + F), s3 = ldcg4(sr + 2 * F);
            const float4 gq = ldcg4(s.g0 + a * F + c);
            const float* gm = s.g2 + a * 3 * F + c;
            const float4 g0 = ldcg4(gm), g1 = ldcg4(gm + F), g2 = ldcg4(gm + 2 * F);
            const float4 svw = f4_fma(v2, w2, f4_fma(v1, w1, f4_mul(v0, w0)));
            float* gs = s.o0 + a * 3 * F + c;
            st4(gs, gq);
            st4(gs + F, f4_fma(g2, w2, f4_fma(g1, w1, f4_mul(g0, w0))));
            st4(gs + 2 * F, f4_mul(gq, svw));
            const float4 gqs3 = f4_mul(gq, s3);
            float* gvw = s.o1 + a * 6 * F + c;
            st4(gvw, f4_mul(gqs3, w0));
            st4(gvw + F, f4_fma(g0, s2, f4_mul(gqs3, v0)));
            st4(gvw + 2 * F, f4_mul(gqs3, w1));
            st4(gvw + 3 * F, f4_fma(g1, s2, f4_mul(gqs3, v1)));
            st4(gvw + 4 * F, f4_mul(gqs3, w2));
            st4(gvw + 5 * F, f4_fma(g2, s2, f4_mul(gqs3, v2)));
        }
    } else if (s.kind == SPK_CHAIN_MIX_CTX_BWD) {   // g0 = g_ctx [N,2F], g1 = VW, g2 = g_q -> o0 = g_q', o1 = g_VW (V third +=)
#pragma unroll 1
        GLUE_LOOP_BEGIN
            const float* v = s.g1 + a * 6 * F + c;
            const float4 v0 = ldcg4(v), v1 = ldcg4(v + 2 * F), v2 = ldcg4(v + 4 * F);
            const float4 gc = ldcg4(s.g0 + a * 2 * F + c), gn0 = ldcg4(s.g0 + a * 2 * F + F + c);
            const float4 gq = ldcg4(s.g2 + a * F + c);
            float* gv = s.o1 + a * 6 * F + c;
            const float4 o0 = ldcg4(gv), o1 = ldcg4(gv + 2 * F), o2 = ldcg4(gv + 4 * F);
            const float4 nn = f4_fma(v2, v2, f4_fma(v1, v1, f4_mul(v0, v0)));
            const float4 gn = make_float4(gn0.x / sqrtf(nn.x + s.eps), gn0.y / sqrtf(nn.y + s.eps),
                                          gn0.z / sqrtf(nn.z + s.eps), gn0.w / sqrtf(nn.w + s.eps));
            st4(s.o0 + a * F + c, f4_add(gq, gc));
            st4(gv, f4_fma(gn, v0, o0));
            st4(gv + 2 * F, f4_fma(gn, v1, o1));
            st4(gv + 4 * F, f4_fma(gn, v2, o2));
        }
    }
}

__global__ void __launch_bounds__(NTHREADS, 1) k_atom_chain(const __grid_constant__ ChainArgs g) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ __align__(8) uint64_t full_bar[NST];
    __shared__ __align__(8) uint64_t empty_bar[NST];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NST; ++s) {
            mbar_init(&full_bar[s], 2);      // expect_tx arrive (weight TMA) + arrive after the A tile is stored
            mbar_init(&empty_bar[s], N_CONS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    SPK_PDL_WAIT();

    // step-major item numbering
    int base[SPK_CHAIN_MAX_STEPS + 1];
    base[0] = 0;
#pragma unroll
    for (int s = 0; s < SPK_CHAIN_MAX_STEPS; ++s)
        base[s + 1] = base[s] + (s < g.n_steps ? items_per_tile(g.step[s]) * g.n_tiles : 0);
    const int total = base[g.n_steps];

    uint32_t ktg = 0;            // K-tiles this CTA has pushed through the pipeline so far (same value in every warp)
    __shared__ int s_item;
    int* const next_item = g.ws + g.n_steps * g.n_tiles + 1;
    for (;;) {
        // ---- claim the next item (dynamic, in increasing order: the lowest unfinished item is always held by a RESIDENT
        // CTA, so the dependency spin below cannot deadlock even if fewer CTAs than launched are co-resident) and wait
        // until every item of the previous step for its atom tile has been published
        if (tid == 0) {
            const int it = atomicAdd(next_item, 1);
            if (g.trace && it < total) g.trace[(int64_t)it * 8 + 0] = gtime();      // claimed
            if (it < total) {
                int sj = 0;
                while (it >= base[sj + 1]) ++sj;
                if (sj > 0) {
                    const int ipt_prev = items_per_tile(g.step[sj - 1]);
                    const int tile_j = (it - base[sj]) / items_per_tile(g.step[sj]);
                    const int* flag = g.ws + (sj - 1) * g.n_tiles + tile_j;
                    while (ld_acquire(flag) < ipt_prev) __nanosleep(20);
                }
            }
            s_item = it;
        }
        __syncthreads();
        const int item = s_item;
        if (item >= total) break;
        int si = 0;
        while (item >= base[si + 1]) ++si;
        const spk_chain_step_t& st = g.step[si];
        const int ipt = items_per_tile(st);
        const int local = item - base[si];
        const int tile = local / ipt, sub = local - tile * ipt;
        const int64_t a0 = (int64_t)tile * TM;
        const int64_t a1 = min(a0 + TM, g.n_atoms);
        CTRACE(1, gtime());                                                          // dependencies satisfied
        CTRACE(4, (long long)blockIdx.x);
        CTRACE(5, (long long)si);
        CTRACE(6, (long long)tile);

        if (st.kind != SPK_CHAIN_GEMM) {
            glue_item(st, a0, a1, tid);
        } else {
            const int ncol = st.N / TN;
            const int rsub = sub / ncol, col = sub - rsub * ncol;
            const int64_t M = g.n_atoms * st.rows_per_atom;
            const int64_t m0 = ((int64_t)tile * st.rows_per_atom + rsub) * TM;
            const int n0 = col * TN;
            const int nk = st.K / TK;
            const bool live = m0 < M;            // rows of a partial last atom tile may leave whole row tiles empty
            if (live) {
                if (warp >= W_PROD0) {
                    // =========================================== producers ===========================================
                    const int chunk = lane & 3, rsubr = lane >> 2;
                    const float* wp_tile0 = st.Wp + (int64_t)col * nk * (2 * OPER_B / 4);
                    const int pw = warp - W_PROD0;
                    // K-tile kt of this item has global number ktg + kt and belongs to producer (ktg + kt) % NPROD
                    int kt = (int)((pw + NPROD - (ktg % NPROD)) % NPROD);
                    for (; kt < nk; kt += NPROD) {
                        const uint32_t gk = ktg + kt;
                        const int s = gk % NST;
                        const uint32_t use = gk / NST;
                        uint8_t* stg = smem + s * STAGE_BYTES;
                        const int k = kt * TK + chunk * 4;
                        // every load unconditional (clamped row, zeroed afterwards) and the a_pre variant chosen by a
                        // warp-uniform branch OUTSIDE the batch: loads under a data-dependent branch are serialised by
                        // the compiler
                        float4 av[16];
                        const int64_t m_last = M - 1;
#pragma unroll
                        for (int p = 0; p < 16; ++p) {
                            const int64_t m = m0 + p * 8 + rsubr;
                            av[p] = ldcg4(st.A + (m < M ? m : m_last) * st.lda + k);
                        }
                        if (st.a_pre) {              // a_pre holds act'(pre) saved by the forward layer (SPK_ACT_GIVEN)
#pragma unroll
                            for (int h = 0; h < 2; ++h) {            // two batches of 8: 16 more float4 would spill
                                float4 dv[8];
#pragma unroll
                                for (int p = 0; p < 8; ++p) {
                                    const int64_t m = m0 + (h * 8 + p) * 8 + rsubr;
                                    dv[p] = ldcg4(st.a_pre + (m < M ? m : m_last) * st.lda + k);
                                }
#pragma unroll
                                for (int p = 0; p < 8; ++p) {
                                    float4& v = av[h * 8 + p];
                                    v.x *= dv[p].x; v.y *= dv[p].y; v.z *= dv[p].z; v.w *= dv[p].w;
                                }
                            }
                        }
#pragma unroll
                        for (int p = 0; p < 16; ++p)
                            if (m0 + p * 8 + rsubr >= M) av[p] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (use >= 1) mbar_wait(&empty_bar[s], (use - 1) & 1);
                        if (lane == 0) {
                            mbar_expect_tx(&full_bar[s], 2 * OPER_B);
                            tma_load(stg + 2 * OPER_A, wp_tile0 + (int64_t)kt * (2 * OPER_B / 4), 2 * OPER_B, &full_bar[s]);
                        }
#pragma unroll
                        for (int p = 0; p < 16; ++p) {
                            const float4 v = av[p];
                            float4 hi, lo;
                            hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
                            lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
                            const int off = tile_off(p * 8 + rsubr, chunk);
                            *reinterpret_cast<float4*>(stg + off) = hi;
                            *reinterpret_cast<float4*>(stg + OPER_A + off) = lo;
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&full_bar[s]);
                    }
                } else {
                    // =========================================== consumers: wgmma ===========================================
                    const int wg = warp >> 2;
                    float acc[NB][32];
#pragma unroll
                    for (int cb = 0; cb < NB; ++cb)
#pragma unroll
                        for (int i = 0; i < 32; ++i) acc[cb][i] = 0.f;
                    for (int kt = 0; kt < nk; ++kt) {
                        const uint32_t gk = ktg + kt;
                        const int s = gk % NST;
                        mbar_wait(&full_bar[s], (gk / NST) & 1);
                        const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
                        wg_ktile_3xtf32<NB>(acc, sa + wg * SPK_WG_ROWS_BYTES, sa + OPER_A + wg * SPK_WG_ROWS_BYTES,
                                            sa + 2 * OPER_A, sa + 2 * OPER_A + OPER_B);
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&empty_bar[s]);
                    }
                    // every wgmma of both warpgroups has completed and the producers are done with this item: the stages
                    // now stage the raw fp32 tile for the CTA-wide epilogue
                    wg_bar(1, N_CONS * 32);
                    const int t = tid & 127;
#pragma unroll
                    for (int cb = 0; cb < NB; ++cb)
#pragma unroll
                        for (int i = 0; i < 32; i += 2)
                            *reinterpret_cast<float2*>(reinterpret_cast<float*>(smem) + (wg * 64 + wg_frag_row(t, i)) * EP_LD +
                                                       cb * 64 + wg_frag_col(t, i)) = make_float2(acc[cb][i], acc[cb][i + 1]);
                }
                ktg += nk;
            }
            __syncthreads();
            CTRACE(2, gtime());                                                      // K-loop done, tile staged
            if (live) {
                // =========================================== epilogue: all warps, coalesced ===========================================
                // thread -> fixed group of 4 columns (NTHREADS is a multiple of TN / 4), rows tid / 32 + 15 i
                const float* ept = reinterpret_cast<const float*>(smem);
                const int act = st.act;
                constexpr int RSTEP = NTHREADS / (TN / 4);                   // 15 rows between a thread's elements
                const int c4 = tid % (TN / 4);
                const int n = n0 + c4 * 4;
                float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
                if (st.bias) bv = *reinterpret_cast<const float4*>(st.bias + n);
#pragma unroll 2
                for (int row = tid / (TN / 4); row < TM; row += RSTEP) {
                    const int64_t m = m0 + row;
                    if (m >= M) break;
                    float4 v = *reinterpret_cast<const float4*>(ept + row * EP_LD + c4 * 4);
                    v.x += bv.x; v.y += bv.y; v.z += bv.z; v.w += bv.w;
                    if (act != SPK_ACT_NONE) {
                        float4 d;
                        chain_act_both(v.x, act, v.x, d.x);
                        chain_act_both(v.y, act, v.y, d.y);
                        chain_act_both(v.z, act, v.z, d.z);
                        chain_act_both(v.w, act, v.w, d.w);
                        if (st.y_pre) *reinterpret_cast<float4*>(st.y_pre + m * st.ldy + n) = d;   // act'(pre) for the reverse sweep
                    }
                    if (st.addend) {
                        const float4 a = ldcg4(st.addend + m * st.ld_add + n);
                        v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
                    }
                    *reinterpret_cast<float4*>(st.Y + m * st.ldy + n) = v;
                }
            }
        }
        // ---- publish: all of this item's global writes, then one increment of the (step, tile) counter
        __syncthreads();
        if (tid == 0) {
            __threadfence();
            atomicAdd(g.ws + si * g.n_tiles + tile, 1);
        }
        CTRACE(3, gtime());                                                          // published
    }

    // ---- the last CTA to finish resets the counters for the next launch (the workspace has to be zero only once)
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        int* fin = g.ws + g.n_steps * g.n_tiles;
        const int prev = atomicAdd(fin, 1);
        if (prev == (int)gridDim.x - 1) {
            for (int i = 0; i < g.n_steps * g.n_tiles; ++i) g.ws[i] = 0;
            *fin = 0;
            *next_item = 0;
            __threadfence();
        }
    }
}

}  // namespace

extern "C" size_t spk_atom_chain_workspace_ints(int n_steps, int64_t n_atoms) {
    return (size_t)n_steps * (size_t)spk_cdiv(n_atoms, TM) + 2;
}

extern "C" int spk_atom_chain_debug(const spk_chain_step_t* steps, int n_steps, int64_t n_atoms, int32_t* workspace,
                                    size_t workspace_ints, int flags, long long* trace, spk_stream_t stream);

extern "C" int spk_atom_chain(const spk_chain_step_t* steps, int n_steps, int64_t n_atoms, int32_t* workspace,
                              size_t workspace_ints, int flags, spk_stream_t stream) {
    return spk_atom_chain_debug(steps, n_steps, n_atoms, workspace, workspace_ints, flags, nullptr, stream);
}

// same launch with per-item time stamps (8 x int64 per item: claimed, dependencies satisfied, K-loop done, published [ns,
// %globaltimer], CTA, step, atom tile, -) written to `trace` (device, >= 8 * items int64) -- development aid
extern "C" int spk_atom_chain_debug(const spk_chain_step_t* steps, int n_steps, int64_t n_atoms, int32_t* workspace,
                                    size_t workspace_ints, int flags, long long* trace, spk_stream_t stream) {
    if (!steps || n_steps <= 0 || n_steps > SPK_CHAIN_MAX_STEPS || n_atoms < 0 || !workspace) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (n_atoms > (1ll << 31) - 256) return SPK_ERR_UNSUPPORTED;
    if (workspace_ints < spk_atom_chain_workspace_ints(n_steps, n_atoms)) return SPK_ERR_ARG;
    ChainArgs g;
    g.n_steps = n_steps;
    g.n_atoms = n_atoms;
    g.n_tiles = (int)spk_cdiv(n_atoms, TM);
    g.ws = workspace;
    g.trace = trace;
    auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    int64_t items = 0;
    for (int s = 0; s < n_steps; ++s) {
        const spk_chain_step_t& st = steps[s];
        g.step[s] = st;
        if (st.kind == SPK_CHAIN_GEMM) {
            if (st.rows_per_atom < 1 || st.K <= 0 || st.N <= 0 || !st.A || !st.Wp || !st.Y) return SPK_ERR_ARG;
            if ((st.K % TK) || (st.N % TN) || (st.lda & 3) || (st.ldy & 3) || (st.ld_add & 3)) return SPK_ERR_UNSUPPORTED;
            if (st.lda < st.K || st.ldy < st.N || (st.addend && st.ld_add < st.N)) return SPK_ERR_ARG;
            if (st.act < 0 || st.act > 2) return SPK_ERR_ARG;
            if (!(al(st.A) && al(st.a_pre) && al(st.Wp) && al(st.bias) && al(st.addend) && al(st.Y) && al(st.y_pre)))
                return SPK_ERR_UNSUPPORTED;
            items += (int64_t)st.rows_per_atom * (st.N / TN) * g.n_tiles;
        } else if (st.kind >= SPK_CHAIN_MIX_CTX && st.kind <= SPK_CHAIN_MIX_CTX_BWD) {
            if (st.F <= 0 || (st.F & 3) || !st.g0 || !st.g1 || !st.o0) return SPK_ERR_ARG;
            if (st.kind != SPK_CHAIN_MIX_CTX && (!st.g2 || !st.o1)) return SPK_ERR_ARG;
            if ((st.kind == SPK_CHAIN_MIX_UPDATE || st.kind == SPK_CHAIN_MIX_UPDATE_BWD) && !st.g3) return SPK_ERR_ARG;
            if (!(al(st.g0) && al(st.g1) && al(st.g2) && al(st.g3) && al(st.o0) && al(st.o1))) return SPK_ERR_UNSUPPORTED;
            items += g.n_tiles;
        } else {
            return SPK_ERR_ARG;
        }
    }
    if (items >= (1ll << 31)) return SPK_ERR_UNSUPPORTED;
    // SPK_CHAIN_FLAG_NFOLD selects nothing here: with register accumulators both accumulation schemes of the 3xTF32
    // products are the same fresh-accumulator-per-K-tile scheme (wg_ktile_3xtf32)
    (void)flags;
    static SpkSmemOnce once;
    if (cudaError_t e = once.set(k_atom_chain, SMEM_BYTES); e != cudaSuccess) return SPK_CUDA_ERR(e);
    int64_t nb = spk_num_sms();                       // one persistent CTA per SM
    if (nb > items) nb = items;
    spk_launch(k_atom_chain, (unsigned)nb, NTHREADS, SMEM_BYTES, spk_st(stream), g);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

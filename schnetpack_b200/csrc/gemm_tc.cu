// Dense layer on the Hopper tensor cores (wgmma, register accumulators) with 3xTF32 error compensation:
//
//     Y = act( (A .* act'(a_pre)) * W^T + bias ) + addend            A [M,K] fp32, W [N,K] fp32 (K contiguous)
//
// The reference computes these layers with true-fp32 cuBLAS SGEMM (torch matmul precision "highest"); single-pass TF32
// would miss the 1e-5 parity bar by two orders of magnitude.  Scheme (DESIGN.md section 3):
//   * every operand is split  x = hi + lo  (hi = round-to-nearest TF32, lo = x - hi exact in fp32); three tensor-core
//     products Ah*Bh + Al*Bh + Ah*Bl are formed (Al*Bl is O(2^-24));
//   * the tensor core adds into its accumulator with TRUNCATION, which biases long K-sums toward zero.  Therefore the products
//     of each K-tile (16 floats = 2 k-steps) go into a FRESH accumulator that is added to the fp32 running sum with IEEE
//     round-to-nearest (wg_ktile_3xtf32, wgmma.cuh).
//
// Warp-specialised pipeline, one CTA per 128 x TN output tile:
//   warps 8-11  producers: K-tile kt belongs to warp kt % NPROD and stage kt % NST (NPROD divides NST).  Lane 0 arms
//               full[stage] with the byte count of the weight tile and issues ONE TMA bulk copy (cp.async.bulk) of the
//               pre-packed W_hi|W_lo operand tile (the weights are static, so the host packs them once in the exact
//               shared-memory operand layout, spk_tc_pack_weight); all lanes load the A tile with coalesced 128-bit loads
//               (optional backward prologue x act'(a_pre)), split hi/lo in registers and st.shared it K-major with the
//               64-byte swizzle (row = 64 B, 8-row atoms of 512 B, 16 B chunk index XOR row bits [1,3));
//               fence.proxy.async; arrive on full[stage];
//   warps 0-7   two consumer warpgroups, rows 0-63 and 64-127 of the tile: wait full[stage], issue the stage's wgmma
//               (m64n64k8, one commit group per 64-column block), add each completed group to the register sum while
//               the next one runs, arrive on empty[stage]; after the last K-tile the raw tile is staged in shared
//               memory (the pipeline stages are free by then);
//   all warps   epilogue: bias / activation (+ saved derivative) / addend / stores, 16 B per thread, whole 128 B lines
//               per row segment.
#include "wgmma.cuh"

namespace {

constexpr int TM = 128;                        // rows per CTA tile (two m64 warpgroups)
constexpr int TK = 16;                         // floats per K-tile = 2 k-steps
constexpr int N_CONS = 8;                      // consumer warps 0-7 (two warpgroups)
constexpr int W_PROD0 = 8;
constexpr int OPER_A = TM * TK * 4;            // 8192 B: A tile, K-major, SWIZZLE_64B
#ifndef SPK_TC_STAGGER
#define SPK_TC_STAGGER 300
#endif

template <int TN>
struct Cfg {
    static constexpr int NST = TN == 64 ? 8 : 4;           // shared-memory stages (8 x 32 KB would not fit at TN = 128)
    static constexpr int NPROD = 4;                         // producer warps; NPROD divides NST, so all uses of a stage belong
                                                            // to ONE warp and are strictly ordered (a parity wait cannot
                                                            // tell phase u from phase u+2).  384 threads leave the
                                                            // consumers' sum and two fresh accumulators (128 floats at
                                                            // TN = 128) room in registers without spills
    static constexpr int OPER_B = TN * TK * 4;              // weight tile, same layout as the A tile
    static constexpr int STAGE_BYTES = 2 * OPER_A + 2 * OPER_B;   // A_hi, A_lo, W_hi, W_lo
    static constexpr int EP_LD = TN + 4;                    // padded row of the epilogue staging tile (floats)
    static constexpr int SMEM_BYTES = NST * STAGE_BYTES + 1024;   // + slack to align the stages to 1024 B
    static constexpr int NTHREADS = (W_PROD0 + NPROD) * 32;
    static constexpr int NB = TN / 64;                      // m64n64 column blocks per consumer warpgroup
    static_assert(NST * STAGE_BYTES >= TM * EP_LD * 4, "epilogue staging tile reuses the pipeline stages");
    static_assert(NST % NPROD == 0, "a stage must be owned by exactly one producer warp");
};

// raw accumulator fragments of a consumer warpgroup (rows wg*64..) -> row-major fp32 staging tile with rows of ld floats
template <int NB>
__device__ __forceinline__ void wg_stage_tile(const float (&acc)[NB][32], float* ep, int ld, int wg, int t) {
#pragma unroll
    for (int cb = 0; cb < NB; ++cb)
#pragma unroll
        for (int i = 0; i < 32; i += 2)
            *reinterpret_cast<float2*>(ep + (wg * 64 + wg_frag_row(t, i)) * ld + cb * 64 + wg_frag_col(t, i)) =
                make_float2(acc[cb][i], acc[cb][i + 1]);
}

// activation-gradient helper kept out of line: the producer loop is fully unrolled over a register array, inlining
// expf/log1pf 16x blew the kernel up and it stalled on the instruction cache (ncu: stall_no_inst 30 %)
template <int ACT>
__device__ __noinline__ float4 act_grad4(float4 q) {
    return make_float4(spk_act_grad(q.x, ACT), spk_act_grad(q.y, ACT), spk_act_grad(q.z, ACT), spk_act_grad(q.w, ACT));
}

struct TcArgs {
    const float* A;
    const float* a_pre;
    const float* Wp;   // packed weights: [ceil(N/TN)][ceil(K/16)][W_hi tile | W_lo tile] in operand layout
    const float* bias;
    const float* addend;
    float* Y;
    float* y_pre;
    int64_t M, lda, ld_add, ldy;
    int K, N, a_act, act, save_deriv;
};


// Column-tile width.  A weight with N % 128 == 0 is packed in BOTH tile widths (the layouts differ); the launch picks 128
// when N >= 256 or when 64-wide tiles would need more than one wave of CTAs (M = 3 x atoms in the mu channel mix).
__host__ __device__ __forceinline__ bool has_wide(int N) { return N % 128 == 0; }
__host__ __device__ __forceinline__ size_t packed_floats_tn(int N, int K, int TN) {
    return (size_t)((N + TN - 1) / TN) * ((K + TK - 1) / TK) * (2 * TN * TK);
}
static inline int tile_n(int64_t M, int N) {
#ifdef TC_FORCE_TN
    return TC_FORCE_TN;
#else
    if (!has_wide(N)) return 64;
    if (N >= 256) return 128;
    return spk_cdiv(M, TM) * (N / 64) > spk_num_sms() ? 128 : 64;
#endif
}

// one-time packing of a weight matrix W [N,K] into per-(n-tile, k-tile) operand tiles [hi | lo]
__global__ void k_pack_weight(const float* __restrict__ W, int N, int K, int TN, float* __restrict__ out) {
    SPK_PDL_WAIT_ONLY();
    const int nkt = (K + TK - 1) / TK;
    const int64_t total = (int64_t)((N + TN - 1) / TN) * nkt * TN * TK;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int kk = (int)(t % TK);
    const int r = (int)((t / TK) % TN);
    const int kt = (int)((t / (TK * TN)) % nkt);
    const int nt = (int)(t / ((int64_t)TK * TN * nkt));
    const int n = nt * TN + r, k = kt * TK + kk;
    const float w = (n < N && k < K) ? W[(int64_t)n * K + k] : 0.f;
    const float hi = tf32_rn(w), lo = w - hi;
    const int oper_b = TN * TK;                               // floats per operand tile
    float* tile = out + ((int64_t)nt * nkt + kt) * (2 * oper_b);
    const int off = tile_off(r, kk >> 2) / 4 + (kk & 3);
    tile[off] = hi;
    tile[oper_b + off] = lo;
}

// Fast-path requirements (checked by the dispatcher, otherwise the fp32 kernel runs): lda, ldy, ld_add, K, N multiples of 4
// and 16 B-aligned base pointers.
template <int TN, int A_ACT, int ACT>
__global__ void __launch_bounds__(Cfg<TN>::NTHREADS, 1) k_dense_tc(TcArgs g) {
    using C = Cfg<TN>;
    constexpr int NST = C::NST, NPROD = C::NPROD, OPER_B = C::OPER_B, STAGE_BYTES = C::STAGE_BYTES, EP_LD = C::EP_LD,
                  NTHREADS = C::NTHREADS, NB = C::NB;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    __shared__ __align__(8) uint64_t full_bar[NST];
    __shared__ __align__(8) uint64_t empty_bar[NST];

    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    const int64_t m0 = (int64_t)blockIdx.x * TM;
    const int n0 = blockIdx.y * TN;
    const int nk = (g.K + TK - 1) / TK;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NST; ++s) {
            mbar_init(&full_bar[s], 2);      // expect_tx arrive (weight TMA) + arrive after the A tile is stored
            mbar_init(&empty_bar[s], N_CONS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // the weight tiles of the first NST K-tiles are static operands: their TMA copies are issued here, BEFORE
        // griddepcontrol.wait, and land while the previous kernel is still running (pack kernels never trigger their
        // dependents early, common.cuh); after the wait only the A tiles remain to be fetched
        const float* wp0 = g.Wp + (int64_t)blockIdx.y * nk * (2 * OPER_B / 4);
        for (int s = 0; s < NST && s < nk; ++s) {
            mbar_expect_tx(&full_bar[s], 2 * OPER_B);
            tma_load(smem + s * STAGE_BYTES + 2 * OPER_A, wp0 + (int64_t)s * (2 * OPER_B / 4), 2 * OPER_B, &full_bar[s]);
        }
    }
    __syncthreads();
    SPK_PDL_WAIT();      // barrier init above overlaps the previous kernel's tail; no global access yet

    if (warp >= W_PROD0) {
        // =========================================== producers ===========================================
        const int chunk = lane & 3, rsub = lane >> 2;          // 4 x 16 B chunks per row, 8 rows per pass, 16 passes
        const float* wp_tile0 = g.Wp + (int64_t)blockIdx.y * nk * (2 * OPER_B / 4);
        for (int kt = warp - W_PROD0; kt < nk; kt += NPROD) {
            const int s = kt % NST, use = kt / NST;
            uint8_t* st = smem + s * STAGE_BYTES;
            const int k = kt * TK + chunk * 4;
            const bool k_ok = k < g.K;                         // K % 4 == 0: a 16 B chunk is entirely in or out
#if SPK_TC_STAGGER > 0
            // The first NPROD K-tiles are requested in K order, SPK_TC_STAGGER cycles apart: issued all at once they share
            // the SM's L2 port and K-tile 0 -- which the first MMA waits for -- lands last as likely as first.
            if (kt < NPROD && kt > 0) {
                const long long t0 = clock64();
                while (clock64() - t0 < (long long)kt * SPK_TC_STAGGER) { }
            }
#endif
            // ---- issue the global loads first (latency overlaps the wait for the stage) ----
            float4 av[16];
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                const int64_t m = m0 + p * 8 + rsub;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (k_ok && m < g.M) {
                    v = *reinterpret_cast<const float4*>(g.A + m * g.lda + k);
                    if (A_ACT == SPK_ACT_GIVEN) {          // a_pre holds act'(pre) saved by the forward layer
                        const float4 d = *reinterpret_cast<const float4*>(g.a_pre + m * g.lda + k);
                        v.x *= d.x; v.y *= d.y; v.z *= d.z; v.w *= d.w;
                    } else if (A_ACT != SPK_ACT_NONE) {
                        const float4 d = act_grad4<A_ACT>(*reinterpret_cast<const float4*>(g.a_pre + m * g.lda + k));
                        v.x *= d.x; v.y *= d.y; v.z *= d.z; v.w *= d.w;
                    }
                }
                av[p] = v;
            }
            if (use >= 1) mbar_wait(&empty_bar[s], (use - 1) & 1);      // wgmma that read this stage have completed
            if (lane == 0 && use >= 1) {   // weight tile (hi|lo, operand layout): one TMA bulk copy (first uses: prefetched above)
                mbar_expect_tx(&full_bar[s], 2 * OPER_B);
                tma_load(st + 2 * OPER_A, wp_tile0 + (int64_t)kt * (2 * OPER_B / 4), 2 * OPER_B, &full_bar[s]);
            }
#pragma unroll
            for (int p = 0; p < 16; ++p) {
                const float4 v = av[p];
                float4 hi, lo;
                hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
                lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
                const int off = tile_off(p * 8 + rsub, chunk);
                *reinterpret_cast<float4*>(st + off) = hi;
                *reinterpret_cast<float4*>(st + OPER_A + off) = lo;
            }
            // generic-proxy stores -> visible to the tensor core (async proxy), then signal the consumers
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[s]);
            if (lane == 0 && (kt == 0 || kt == nk - 1)) SPK_TL_PHASE(kt == 0 ? 2 : 3);   // first / last stage published
        }
    } else {
        // =========================================== consumers: wgmma, fp32 accumulation in registers ===========================
        // The work is a sequence of units u = (K-tile u / NB, column block u % NB), each one wgmma group into a fresh
        // accumulator.  Two fresh accumulators alternate: unit u + 1 is on the tensor core while unit u is added to its
        // column block's sum, so the tensor core is not drained between units.  Each column block still receives its
        // K-tiles in ascending order, one fresh accumulator per K-tile (the numerics of wg_ktile_3xtf32).
        const int wg = warp >> 2;                        // rows wg * 64 .. wg * 64 + 63 of the tile
        float acc[NB][32], t0[32], t1[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
#pragma unroll
            for (int cb = 0; cb < NB; ++cb) acc[cb][i] = 0.f;
            t0[i] = t1[i] = 0.f;                         // defined operands; each unit's first product overwrites them
        }
        const int nu = nk * NB;
        auto issue = [&](float (&t)[32], int u) {
            const int kt = u / NB, cb = u % NB, s = kt % NST;
            if (cb == 0) mbar_wait(&full_bar[s], (kt / NST) & 1);
            const uint32_t sa = smem_u32(smem + s * STAGE_BYTES), bo = (uint32_t)(cb * SPK_WG_ROWS_BYTES);
            wg_ktile_3xtf32_issue(t, sa + wg * SPK_WG_ROWS_BYTES, sa + OPER_A + wg * SPK_WG_ROWS_BYTES,
                                  sa + 2 * OPER_A + bo, sa + 2 * OPER_A + OPER_B + bo);
        };
        auto retire = [&](const float (&t)[32], float (&a)[32], int u) {   // unit u has completed
#pragma unroll
            for (int i = 0; i < 32; ++i) a[i] += t[i];
            const int kt = u / NB;
            if (u % NB == NB - 1) {                      // every wgmma that read this K-tile's stage has completed
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[kt % NST]);
                if (warp == 0 && lane == 0 && (kt == 0 || kt == nk - 1)) SPK_TL_PHASE(kt == 0 ? 4 : 5);
            }
        };
        // u is even: t0 holds column block 0 and t1 column block NB - 1 (both block 0 when NB == 1).  The loop body issues
        // unconditionally (a conditional issue makes ptxas serialise every wgmma of the kernel); the tail is peeled.
        issue(t0, 0);
        int u = 0;
        for (; u + 2 < nu; u += 2) {
            issue(t1, u + 1);
            wgmma_wait<1>();
            retire(t0, acc[0], u);
            issue(t0, u + 2);
            wgmma_wait<1>();
            retire(t1, acc[NB - 1], u + 1);
        }
        if (u + 1 < nu) {
            issue(t1, u + 1);
            wgmma_wait<1>();
            retire(t0, acc[0], u);
            wgmma_wait<0>();
            retire(t1, acc[NB - 1], u + 1);
        } else {
            wgmma_wait<0>();
            retire(t0, acc[0], u);
        }
        // both warpgroups have completed every wgmma (and the producers every store): the stages now hold the raw tile
        wg_bar(1, N_CONS * 32);
        wg_stage_tile<NB>(acc, reinterpret_cast<float*>(smem), EP_LD, wg, tid & 127);
        if (warp == 0 && lane == 0) SPK_TL_PHASE(6);
    }
    __syncthreads();
    // =========================================== epilogue: all warps, coalesced ===========================================
    {
        // Every thread owns ONE float4 column group (NTHREADS is a multiple of TN / 4) and walks down the rows: the bias is
        // loaded once, pointers advance by constant strides, and the loads of RB rows are issued before their stores (the
        // outputs may alias the inputs as far as the compiler knows, so it cannot hoist them itself).
        static_assert(NTHREADS % (TN / 4) == 0, "one column group per thread");
        constexpr int RSTEP = NTHREADS / (TN / 4), RB = 3;
        const float* ept = reinterpret_cast<const float*>(smem);
        const int c4 = tid % (TN / 4);
        const int n = n0 + c4 * 4;
        const int rows_here = (int)(g.M - m0 < TM ? g.M - m0 : TM);
        if (n < g.N) {                                           // N % 4 == 0: whole float4 groups only
            float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g.bias) bv = *reinterpret_cast<const float4*>(g.bias + n);
            const bool deriv = g.y_pre && g.save_deriv && ACT != SPK_ACT_NONE;
#pragma unroll 1
            for (int row0 = tid / (TN / 4); row0 < rows_here; row0 += RSTEP * RB) {
                float4 v[RB], ad[RB];
#pragma unroll
                for (int e = 0; e < RB; ++e) {
                    const int row = row0 + e * RSTEP;
                    v[e] = ad[e] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (row < rows_here) {
                        v[e] = *reinterpret_cast<const float4*>(ept + row * EP_LD + c4 * 4);
                        if (g.addend) ad[e] = *reinterpret_cast<const float4*>(g.addend + (m0 + row) * g.ld_add + n);
                    }
                }
#pragma unroll
                for (int e = 0; e < RB; ++e) {
                    const int row = row0 + e * RSTEP;
                    if (row >= rows_here) continue;
                    const int64_t o = (m0 + row) * g.ldy + n;
                    float4 x = make_float4(v[e].x + bv.x, v[e].y + bv.y, v[e].z + bv.z, v[e].w + bv.w);
                    if (deriv) {
                        float4 d;
                        spk_act_both(x.x, ACT, x.x, d.x);
                        spk_act_both(x.y, ACT, x.y, d.y);
                        spk_act_both(x.z, ACT, x.z, d.z);
                        spk_act_both(x.w, ACT, x.w, d.w);
                        *reinterpret_cast<float4*>(g.y_pre + o) = d;
                    } else {
                        if (g.y_pre)
                            *reinterpret_cast<float4*>(g.y_pre + o) = g.save_deriv ? make_float4(1.f, 1.f, 1.f, 1.f) : x;
                        if (ACT != SPK_ACT_NONE)
                            x = make_float4(spk_act(x.x, ACT), spk_act(x.y, ACT), spk_act(x.z, ACT), spk_act(x.w, ACT));
                    }
                    x.x += ad[e].x; x.y += ad[e].y; x.z += ad[e].z; x.w += ad[e].w;
                    *reinterpret_cast<float4*>(g.Y + o) = x;
                }
            }
        }
    }
    if (tid == 0) SPK_TL_PHASE(7);                                // this CTA's epilogue stores issued
}

}  // namespace

template <int TN, int A_ACT, int ACT>
static int launch_tc(const TcArgs& g, cudaStream_t st) {
    static SpkSmemOnce once;
    if (cudaError_t e = once.set(k_dense_tc<TN, A_ACT, ACT>, Cfg<TN>::SMEM_BYTES); e != cudaSuccess) return SPK_CUDA_ERR(e);
    dim3 grid((unsigned)spk_cdiv(g.M, TM), (unsigned)spk_cdiv(g.N, TN));
    spk_launch(k_dense_tc<TN, A_ACT, ACT>, grid, Cfg<TN>::NTHREADS, Cfg<TN>::SMEM_BYTES, st, g);
    return 0;
}

template <int TN>
static int dispatch_tc(const TcArgs& g, cudaStream_t st) {
    if (g.a_act == SPK_ACT_NONE)
        return g.act == SPK_ACT_NONE   ? launch_tc<TN, 0, 0>(g, st)
               : g.act == SPK_ACT_SILU ? launch_tc<TN, 0, 1>(g, st)
                                       : launch_tc<TN, 0, 2>(g, st);
    return g.a_act == SPK_ACT_SILU  ? launch_tc<TN, 1, 0>(g, st)
           : g.a_act == SPK_ACT_SSP ? launch_tc<TN, 2, 0>(g, st)
                                    : launch_tc<TN, 3, 0>(g, st);
}

extern "C" size_t spk_tc_packed_floats(int N, int K) {
    return packed_floats_tn(N, K, 64) + (has_wide(N) ? packed_floats_tn(N, K, 128) : 0);
}

extern "C" int spk_tc_pack_weight(const float* W, int N, int K, float* packed, spk_stream_t stream) {
    if (N <= 0 || K <= 0 || !W || !packed) return SPK_ERR_ARG;
    for (int TN = 64; TN <= (has_wide(N) ? 128 : 64); TN *= 2) {
        const int64_t total = (int64_t)((N + TN - 1) / TN) * ((K + TK - 1) / TK) * TN * TK;
        float* out = packed + (TN == 128 ? packed_floats_tn(N, K, 64) : 0);     // [64-wide tiles | 128-wide tiles]
        spk_launch(k_pack_weight, (unsigned)spk_cdiv(total, 256), 256, 0, spk_st(stream), W, N, K, TN, out);
    }
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_dense_tc(const float* A, int64_t M, int K, int64_t lda, const float* a_pre, int a_act,
                            const float* W_packed, int N, const float* bias, int act, const float* addend,
                            int64_t ld_add, float* Y, int64_t ldy, float* y_pre, spk_stream_t stream) {
    if (M < 0 || K <= 0 || N <= 0 || lda < K || ldy < N) return SPK_ERR_ARG;
    const int save_deriv = (act & SPK_SAVE_DERIV) ? 1 : 0;
    act &= ~SPK_SAVE_DERIV;
    if (act < 0 || act > 2 || a_act < 0 || a_act > 3) return SPK_ERR_ARG;
    if (M == 0) return SPK_OK;
    if (!A || !W_packed || !Y) return SPK_ERR_ARG;
    if (addend && ld_add < N) return SPK_ERR_ARG;
    if (!a_pre) a_act = SPK_ACT_NONE;
    auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    const bool fast = !(K & 3) && !(N & 3) && !(lda & 3) && !(ldy & 3) && !(ld_add & 3) && al(A) && al(a_pre) &&
                      al(W_packed) && al(bias) && al(addend) && al(Y) && al(y_pre) &&
                      (a_act == SPK_ACT_NONE || act == SPK_ACT_NONE);
    if (!fast) return SPK_ERR_UNSUPPORTED;   // caller falls back to spk_dense (fp32 CUDA-core kernel)
    TcArgs g;
    g.A = A; g.a_pre = a_pre; g.Wp = W_packed; g.bias = bias; g.addend = addend; g.Y = Y; g.y_pre = y_pre;
    g.M = M; g.lda = lda; g.ld_add = ld_add; g.ldy = ldy; g.K = K; g.N = N; g.a_act = a_act; g.act = act; g.save_deriv = save_deriv;
    cudaStream_t st = spk_st(stream);
    int rc;
    if (tile_n(M, N) == 128) {
        g.Wp = W_packed + packed_floats_tn(N, K, 64);
        rc = dispatch_tc<128>(g, st);
    } else {
        rc = dispatch_tc<64>(g, st);
    }
    if (rc) return rc;
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

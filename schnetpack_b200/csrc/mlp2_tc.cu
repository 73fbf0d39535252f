// Two Dense layers as ONE launch on the Hopper tensor cores (wgmma), hidden tile resident in shared memory:
//
//     H = act(A W0^T + b0)            A [M,K1], W0 [128,K1]                (also stored: act'(pre) [M,128] for the reverse pass)
//     Y = H W1^T + b1 [+ addend]      W1 [N2,128]
//
// Reference: every Dense -> Dense pair of the per-atom path -- interatomic_context_net and intraatomic_context_net of PaiNN
// (representation/painn.py of the reference: Dense(F, F, silu) -> Dense(F, 3F)).
//
// Why: a K = 128 k_dense_tc launch pays a launch boundary, a pipeline fill and an epilogue of its own, and for a pair the
// hidden activations make a round trip through L2 in between.  Here a CTA owns a 128-row tile and ONE 128-column tile of the
// final output; it computes the whole hidden tile itself (every column-tile CTA repeats that GEMM, but there is no second
// launch boundary, no hidden-layer store/load, one load phase), writes act(.) hi/lo-split straight into shared memory in the
// wgmma operand layout (K-major, 64-byte swizzle: exactly what the producers of gemm_tc.cu build from global memory), and runs
// the second GEMM from there while the W1 tiles stream through the same TMA ring.  Precision scheme, pipeline roles, operand
// layout and epilogue are those of gemm_tc.cu (3xTF32, fresh accumulator per K-tile added to fp32 registers).  Each consumer
// warpgroup owns 64 rows of both GEMMs, so the hidden rows it writes are exactly the A rows it reads back.
#include "wgmma.cuh"

namespace {

constexpr int TM = 128, TK = 16, TN = 128, HID = 128;
constexpr int N_CONS = 8, W_PROD0 = 8, NST = 3, NPROD = 3;
constexpr int OPER_A = TM * TK * 4;            // 8192 B
constexpr int OPER_B = TN * TK * 4;            // 8192 B
constexpr int STAGE_BYTES = 2 * OPER_A + 2 * OPER_B;       // A_hi, A_lo, W_hi, W_lo
constexpr int NK2 = HID / TK;                  // K-tiles of the second GEMM
constexpr int A2_BYTES = 2 * NK2 * OPER_A;     // hidden operand [hi, lo][k-tile][128 x 16]
constexpr int EP_LD = TN + 4;
constexpr int SMEM_BYTES = NST * STAGE_BYTES + A2_BYTES + 1024;
constexpr int NTHREADS = (W_PROD0 + NPROD) * 32;
constexpr int NB = TN / 64;                    // m64n64 column blocks per consumer warpgroup
static_assert(A2_BYTES >= TM * EP_LD * 4, "the epilogue staging tile reuses the hidden operand");
static_assert(NST == NPROD, "a stage is owned by exactly one producer warp in both phases");
static_assert(NTHREADS % (TN / 4) == 0, "one column group per thread in the epilogue");

struct Mlp2Args {
    const float* A;
    const float* W0p;      // W0 [128,K1] packed in 128-wide tiles: [k-tile][W_hi | W_lo]
    const float* b0;
    const float* W1p;      // W1 [N2,128] packed in 128-wide tiles: [n-tile][k-tile][W_hi | W_lo]
    const float* b1;
    const float* addend;
    float* Y;
    float* h_deriv;        // act'(pre) of the hidden layer [M,128] (written by the CTAs of column tile 0) or NULL
    int64_t M, lda, ldy, ld_add;
    int K1, N2, act;
};

__global__ void __launch_bounds__(NTHREADS, 1) k_mlp2_tc(Mlp2Args g) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t* sA2 = smem + NST * STAGE_BYTES;
    __shared__ __align__(8) uint64_t full_bar[NST];
    __shared__ __align__(8) uint64_t empty_bar[NST];
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // broadcast: the compiler may treat the role index as warp-uniform
    SPK_PDL_LAUNCH_DEPENDENTS();
    const int64_t m0 = (int64_t)blockIdx.x * TM;
    const int n0 = blockIdx.y * TN;
    const int nk1 = (g.K1 + TK - 1) / TK;
    const int nkt = nk1 + NK2;                 // K-tiles of both GEMMs share one running index (stage / accumulator parities)
    const float* w1_tiles = g.W1p + (int64_t)blockIdx.y * NK2 * (2 * OPER_B / 4);

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < NST; ++s) {
            mbar_init(&full_bar[s], 2);      // expect_tx arrive (weight TMA) + arrive after the A tile is stored (phase 2: plain)
            mbar_init(&empty_bar[s], N_CONS);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // static operands: the first W0 tiles are fetched BEFORE griddepcontrol.wait (pack kernels never trigger early)
        for (int s = 0; s < NST && s < nk1; ++s) {
            mbar_expect_tx(&full_bar[s], 2 * OPER_B);
            tma_load(smem + s * STAGE_BYTES + 2 * OPER_A, g.W0p + (int64_t)s * (2 * OPER_B / 4), 2 * OPER_B, &full_bar[s]);
        }
    }
    __syncthreads();
    SPK_PDL_WAIT();

    if (warp >= W_PROD0) {
        // =========================================== producers ===========================================
        const int p = warp - W_PROD0;
        const int chunk = lane & 3, rsub = lane >> 2;          // 4 x 16 B chunks per row, 8 rows per pass, 16 passes
        for (int kt = p; kt < nk1; kt += NPROD) {               // ---- GEMM 1: A tiles from global memory, W0 tiles by TMA
            const int s = kt % NST, use = kt / NST;
            uint8_t* st = smem + s * STAGE_BYTES;
            const int k = kt * TK + chunk * 4;
            const bool k_ok = k < g.K1;
            float4 av[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const int64_t m = m0 + q * 8 + rsub;
                av[q] = (k_ok && m < g.M) ? *reinterpret_cast<const float4*>(g.A + m * g.lda + k)
                                          : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            if (use >= 1) {
                mbar_wait(&empty_bar[s], (use - 1) & 1);
                if (lane == 0) {
                    mbar_expect_tx(&full_bar[s], 2 * OPER_B);
                    tma_load(st + 2 * OPER_A, g.W0p + (int64_t)kt * (2 * OPER_B / 4), 2 * OPER_B, &full_bar[s]);
                }
            }
#pragma unroll
            for (int q = 0; q < 16; ++q) {
                const float4 v = av[q];
                float4 hi, lo;
                hi.x = tf32_rn(v.x); hi.y = tf32_rn(v.y); hi.z = tf32_rn(v.z); hi.w = tf32_rn(v.w);
                lo.x = v.x - hi.x; lo.y = v.y - hi.y; lo.z = v.z - hi.z; lo.w = v.w - hi.w;
                const int off = tile_off(q * 8 + rsub, chunk);
                *reinterpret_cast<float4*>(st + off) = hi;
                *reinterpret_cast<float4*>(st + OPER_A + off) = lo;
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[s]);
            if (lane == 0 && kt == 0) SPK_TL_PHASE(2);           // first operand stage published
        }
        // ---- GEMM 2: only the W1 tiles travel (the A operand is the hidden tile in shared memory)
        int ktg = nk1 + ((p - nk1 % NPROD) + NPROD) % NPROD;    // first running index >= nk1 owned by this warp
        for (; ktg < nkt; ktg += NPROD) {
            const int s = ktg % NST, use = ktg / NST;
            if (use >= 1) mbar_wait(&empty_bar[s], (use - 1) & 1);
            if (lane == 0) {
                mbar_expect_tx(&full_bar[s], 2 * OPER_B);
                tma_load(smem + s * STAGE_BYTES + 2 * OPER_A, w1_tiles + (int64_t)(ktg - nk1) * (2 * OPER_B / 4), 2 * OPER_B,
                         &full_bar[s]);
                mbar_arrive(&full_bar[s]);                      // the arrival an A tile would have made
            }
            __syncwarp();
        }
    } else {
        // =========================================== consumers: wgmma, fp32 accumulation in registers ===========================
        const int wg = warp >> 2, t = tid & 127;         // rows wg * 64 .. wg * 64 + 63 of both GEMMs
        float acc[NB][32];
        auto gemm = [&](int kt_begin, int kt_end) {
#pragma unroll
            for (int cb = 0; cb < NB; ++cb)
#pragma unroll
                for (int i = 0; i < 32; ++i) acc[cb][i] = 0.f;
            for (int kt = kt_begin; kt < kt_end; ++kt) {
                const int s = kt % NST;
                mbar_wait(&full_bar[s], (kt / NST) & 1);
                const uint32_t sa = smem_u32(smem + s * STAGE_BYTES);
                const bool second = kt >= nk1;
                const uint32_t a_hi = second ? smem_u32(sA2 + (kt - nk1) * OPER_A) : sa;
                const uint32_t a_lo = second ? smem_u32(sA2 + (NK2 + kt - nk1) * OPER_A) : sa + OPER_A;
                wg_ktile_3xtf32<NB>(acc, a_hi + wg * SPK_WG_ROWS_BYTES, a_lo + wg * SPK_WG_ROWS_BYTES, sa + 2 * OPER_A,
                                    sa + 2 * OPER_A + OPER_B);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[s]);
            }
        };
        // ---- GEMM 1 -> hidden tile: + b0, activation (value and derivative), hi/lo split into the operand
        gemm(0, nk1);
        SPK_TL_PHASE(3);
#pragma unroll
        for (int cb = 0; cb < NB; ++cb) {
#pragma unroll
            for (int i = 0; i < 32; i += 2) {
                const int row = wg * 64 + wg_frag_row(t, i);
                const int c = cb * 64 + wg_frag_col(t, i);                // hidden unit == K index of GEMM 2 (even)
                float2 bv = make_float2(0.f, 0.f);
                if (g.b0) bv = *reinterpret_cast<const float2*>(g.b0 + c);
                float y0, y1, d0, d1;
                spk_act_both(acc[cb][i] + bv.x, g.act, y0, d0);
                spk_act_both(acc[cb][i + 1] + bv.y, g.act, y1, d1);
                if (g.h_deriv != nullptr && blockIdx.y == 0 && m0 + row < g.M)
                    *reinterpret_cast<float2*>(g.h_deriv + (m0 + row) * HID + c) = make_float2(d0, d1);
                const float h0 = tf32_rn(y0), h1 = tf32_rn(y1);
                const int kt2 = c >> 4, off = tile_off(row, (c & 15) >> 2) + (c & 3) * 4;
                *reinterpret_cast<float2*>(sA2 + kt2 * OPER_A + off) = make_float2(h0, h1);
                *reinterpret_cast<float2*>(sA2 + (NK2 + kt2) * OPER_A + off) = make_float2(y0 - h0, y1 - h1);
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> visible to the tensor core
        wg_bar(1 + wg);                                                   // this warpgroup's hidden rows are complete
        SPK_TL_PHASE(4);
        // ---- GEMM 2 -> raw output tile staged in shared memory once both warpgroups are done reading the hidden operand
        gemm(nk1, nkt);
        wg_bar(3, N_CONS * 32);
#pragma unroll
        for (int cb = 0; cb < NB; ++cb)
#pragma unroll
            for (int i = 0; i < 32; i += 2)
                *reinterpret_cast<float2*>(reinterpret_cast<float*>(sA2) + (wg * 64 + wg_frag_row(t, i)) * EP_LD + cb * 64 +
                                           wg_frag_col(t, i)) = make_float2(acc[cb][i], acc[cb][i + 1]);
        if (warp == 0 && lane == 0) SPK_TL_PHASE(6);              // output tile staged
    }
    __syncthreads();
    // =========================================== epilogue: all warps, coalesced ===========================================
    {
        constexpr int RSTEP = NTHREADS / (TN / 4), RB = 3;
        const float* ept = reinterpret_cast<const float*>(sA2);
        const int c4 = tid % (TN / 4);
        const int n = n0 + c4 * 4;
        const int rows_here = (int)(g.M - m0 < TM ? g.M - m0 : TM);
        if (n < g.N2) {
            float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (g.b1) bv = *reinterpret_cast<const float4*>(g.b1 + n);
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
                    *reinterpret_cast<float4*>(g.Y + (m0 + row) * g.ldy + n) =
                        make_float4(v[e].x + bv.x + ad[e].x, v[e].y + bv.y + ad[e].y, v[e].z + bv.z + ad[e].z,
                                    v[e].w + bv.w + ad[e].w);
                }
            }
        }
    }
    if (tid == 0) SPK_TL_PHASE(7);                                // epilogue stores issued
}

}  // namespace

extern "C" int spk_mlp2_tc(const float* A, int64_t M, int K1, int64_t lda, const float* W0_packed, const float* b0, int act,
                           const float* W1_packed, int N2, const float* b1, const float* addend, int64_t ld_add, float* Y,
                           int64_t ldy, float* h_deriv, spk_stream_t stream) {
    if (M < 0 || K1 <= 0 || N2 <= 0 || lda < K1 || ldy < N2 || act < 0 || act > 2) return SPK_ERR_ARG;
    if (M == 0) return SPK_OK;
    if (!A || !W0_packed || !W1_packed || !Y) return SPK_ERR_ARG;
    if (addend && ld_add < N2) return SPK_ERR_ARG;
    auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    if ((K1 & 3) || (N2 % TN) || (lda & 3) || (ldy & 3) || (ld_add & 3) || !al(A) || !al(W0_packed) || !al(W1_packed) ||
        !al(b0) || !al(b1) || !al(addend) || !al(Y) || !al(h_deriv))
        return SPK_ERR_UNSUPPORTED;            // caller runs the two layers as separate spk_dense_tc launches
    static SpkSmemOnce once;
    if (cudaError_t e = once.set(k_mlp2_tc, SMEM_BYTES); e != cudaSuccess) return SPK_CUDA_ERR(e);
    Mlp2Args g;
    g.A = A; g.W0p = W0_packed; g.b0 = b0; g.W1p = W1_packed; g.b1 = b1; g.addend = addend; g.Y = Y; g.h_deriv = h_deriv;
    g.M = M; g.lda = lda; g.ldy = ldy; g.ld_add = ld_add; g.K1 = K1; g.N2 = N2; g.act = act;
    dim3 grid((unsigned)spk_cdiv(M, TM), (unsigned)(N2 / TN));
    spk_launch(k_mlp2_tc, grid, NTHREADS, SMEM_BYTES, spk_st(stream), g);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

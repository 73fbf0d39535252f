// Dense layer kernel (fp32 FFMA path):  Y = act( (A .* act'(a_pre)) * B + bias ) + addend
// Reference: nn/base.py:52-55 (Dense.forward) and its autograd input-gradient.  True-fp32 accumulation like the
// reference's default torch matmul precision ("highest", cli.py:95-97), so 1e-5 parity holds by construction.
//
// Tiling: BM x 64 output tile per CTA (BM = 128 / 256 threads, or 64 / 128 threads for grids that would not fill the
// chip), BK=16, 8x4 register micro-tile per thread computed as float2 pairs (spk_fma2), A tile stored k-major in shared memory
// so both operand fetches are conflict-free 128-bit LDS; double-buffered shared memory (one barrier per k-tile) with
// the next k-tile prefetched into registers while the current one is multiplied.
#include "common.cuh"

namespace {

constexpr int BN = 64, BK = 16;

struct GemmArgs {
    const float* A;
    const float* a_pre;
    const float* B;
    const float* bias;
    const float* addend;
    float* Y;
    float* y_pre;
    int64_t M, lda, ld_add, ldy;
    int K, N, a_act, act, save_deriv;
};

// activation helpers kept out of line and selected at compile time: inlining the runtime-switched expf/log1pf code into
// the unrolled load / epilogue loops made the kernel 6.3k SASS instructions long and 22 % of its stalls were
// instruction-cache misses
template <int ACT>
__device__ __noinline__ float act_grad1(float q) { return ACT == SPK_ACT_GIVEN ? q : spk_act_grad(q, ACT); }
template <int ACT>
__device__ __noinline__ float act1(float v) { return spk_act(v, ACT); }
template <int ACT>
__device__ __noinline__ float2 act_both1(float v) {
    float y, dy;
    spk_act_both(v, ACT, y, dy);
    return make_float2(y, dy);
}

// BM = 128 (256 threads) for tall problems, BM = 64 / 32 when the 128-row grid would not fill the 132 SMs.
template <int BM, int A_ACT, int ACT>
__global__ void __launch_bounds__(BM * 2) k_dense(GemmArgs g) {
    SPK_PDL_ENTER();
    constexpr int NT = BM * 2;
    constexpr int AS_LD = BM + 4;
    constexpr int A_IT = 2;                       // float4 A loads per thread per k-tile: BM*BK/4 / NT
    __shared__ __align__(16) float As[2][BK][AS_LD];
    __shared__ __align__(16) float Bs[2][BK][BN];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    // global->register staging
    float4 ra[A_IT];
    float4 rb[256 / NT];
    const int a_row = tid >> 2, a_kq = (tid & 3) * 4;  // rows a_row (+ NT/4 per pass), k offset a_kq
    const int b_k = tid >> 4, b_n = (tid & 15) * 4;    // B rows b_k (+ NT/16 per pass)
    const bool a_vec = ((g.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.A) & 15) == 0) &&
                       (!g.a_pre || (reinterpret_cast<uintptr_t>(g.a_pre) & 15) == 0);
    const bool b_vec = ((g.N & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.B) & 15) == 0);

    auto load_tiles = [&](int k0) {
#pragma unroll
        for (int it = 0; it < A_IT; ++it) {
            int64_t m = m0 + a_row + it * (NT / 4);
            int k = k0 + a_kq;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < g.M) {
                const float* p = g.A + m * g.lda + k;
                if (a_vec && k + 3 < g.K) {
                    v = *reinterpret_cast<const float4*>(p);
                    if (A_ACT != SPK_ACT_NONE) {
                        float4 q = *reinterpret_cast<const float4*>(g.a_pre + m * g.lda + k);
                        v.x *= act_grad1<A_ACT>(q.x);
                        v.y *= act_grad1<A_ACT>(q.y);
                        v.z *= act_grad1<A_ACT>(q.z);
                        v.w *= act_grad1<A_ACT>(q.w);
                    }
                } else {
                    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if (k + i < g.K) {
                            t[i] = p[i];
                            if (A_ACT != SPK_ACT_NONE) t[i] *= act_grad1<A_ACT>(g.a_pre[m * g.lda + k + i]);
                        }
                    v = make_float4(t[0], t[1], t[2], t[3]);
                }
            }
            ra[it] = v;
        }
#pragma unroll
        for (int it = 0; it < 256 / NT; ++it) {
            int k = k0 + b_k + it * (NT / 16), n = n0 + b_n;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < g.K) {
                const float* p = g.B + (int64_t)k * g.N + n;
                if (b_vec && n + 3 < g.N) {
                    v = *reinterpret_cast<const float4*>(p);
                } else {
                    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if (n + i < g.N) t[i] = p[i];
                    v = make_float4(t[0], t[1], t[2], t[3]);
                }
            }
            rb[it] = v;
        }
    };
    auto store_tiles = [&](int buf) {
#pragma unroll
        for (int it = 0; it < A_IT; ++it) {
            int r = a_row + it * (NT / 4);
            As[buf][a_kq + 0][r] = ra[it].x;
            As[buf][a_kq + 1][r] = ra[it].y;
            As[buf][a_kq + 2][r] = ra[it].z;
            As[buf][a_kq + 3][r] = ra[it].w;
        }
#pragma unroll
        for (int it = 0; it < 256 / NT; ++it)
            *reinterpret_cast<float4*>(&Bs[buf][b_k + it * (NT / 16)][b_n]) = rb[it];
    };

    // 8x4 micro-tile held as 4x4 float2 accumulators paired along M (spk_fma2: IEEE round-to-nearest per component).
    float2 acc2[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc2[i][j] = make_float2(0.f, 0.f);

    const int nk = (g.K + BK - 1) / BK;
    load_tiles(0);
    store_tiles(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) load_tiles((kt + 1) * BK);      // global loads in flight while this tile is multiplied
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float2 ap[4] = {make_float2(a0.x, a0.y), make_float2(a0.z, a0.w), make_float2(a1.x, a1.y),
                                  make_float2(a1.z, a1.w)};
            const float2 bd[4] = {make_float2(b.x, b.x), make_float2(b.y, b.y), make_float2(b.z, b.z),
                                  make_float2(b.w, b.w)};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc2[i][j] = spk_fma2(ap[i], bd[j], acc2[i][j]);
        }
        if (kt + 1 < nk) store_tiles(buf ^ 1);           // the other buffer was last read before the previous barrier
        __syncthreads();
    }
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            acc[2 * i][j] = acc2[i][j].x;
            acc[2 * i + 1][j] = acc2[i][j].y;
        }

    // epilogue
    const int n = n0 + tx * 4;
    float bv[4] = {0.f, 0.f, 0.f, 0.f};
    if (g.bias) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (n + j < g.N) bv[j] = g.bias[n + j];
    }
    const bool y_vec = ((g.ldy & 3) == 0) && (n + 3 < g.N) && ((reinterpret_cast<uintptr_t>(g.Y) & 15) == 0);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int64_t m = m0 + ty * 8 + i;
        if (m >= g.M) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = acc[i][j] + bv[j];
        if (g.y_pre && g.save_deriv && ACT != SPK_ACT_NONE) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 yd = act_both1<ACT>(v[j]);
                v[j] = yd.x;
                if (n + j < g.N) g.y_pre[m * g.ldy + n + j] = yd.y;
            }
        } else {
            if (g.y_pre) {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (n + j < g.N) g.y_pre[m * g.ldy + n + j] = (g.save_deriv ? 1.0f : v[j]);
            }
            if (ACT != SPK_ACT_NONE) {
#pragma unroll
                for (int j = 0; j < 4; ++j) v[j] = act1<ACT>(v[j]);
            }
        }
        if (g.addend) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (n + j < g.N) v[j] += g.addend[m * g.ld_add + n + j];
        }
        if (y_vec) {
            *reinterpret_cast<float4*>(g.Y + m * g.ldy + n) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (n + j < g.N) g.Y[m * g.ldy + n + j] = v[j];
        }
    }
}

}  // namespace

extern "C" int spk_dense(const float* A, int64_t M, int K, int64_t lda, const float* a_pre, int a_act, const float* B,
                         int N, const float* bias, int act, const float* addend, int64_t ld_add, float* Y, int64_t ldy,
                         float* y_pre, spk_stream_t stream) {
    if (M < 0 || K <= 0 || N <= 0 || lda < K || ldy < N) return SPK_ERR_ARG;
    const int save_deriv = (act & SPK_SAVE_DERIV) ? 1 : 0;
    act &= ~SPK_SAVE_DERIV;
    if (act < 0 || act > 2 || a_act < 0 || a_act > 3) return SPK_ERR_ARG;
    if (M == 0) return SPK_OK;
    if (!A || !B || !Y) return SPK_ERR_ARG;
    if (addend && ld_add < N) return SPK_ERR_ARG;
    GemmArgs g;
    g.A = A; g.a_pre = a_pre; g.B = B; g.bias = bias; g.addend = addend; g.Y = Y; g.y_pre = y_pre;
    g.M = M; g.lda = lda; g.ld_add = ld_add; g.ldy = ldy; g.K = K; g.N = N; g.a_act = a_act; g.act = act; g.save_deriv = save_deriv;
    if (!a_pre) a_act = SPK_ACT_NONE;
    g.a_act = a_act;
    // these layers are skinny (M = atoms): pick the largest row tile that still gives every SM several CTAs, because a
    // CTA's k-loop is a chain of global-load -> shared -> barrier latencies that only co-resident CTAs can hide
    const int64_t want = 3 * (int64_t)spk_num_sms();
    const int64_t nt = spk_cdiv(N, BN);
    const int bm = (spk_cdiv(M, 128) * nt >= want) ? 128 : (spk_cdiv(M, 64) * nt >= want) ? 64 : 32;
    dim3 grid((unsigned)spk_cdiv(M, bm), (unsigned)nt);
    cudaStream_t st = spk_st(stream);
#define LAUNCH_BM(AA, AC)                                                        \
    do {                                                                         \
        if (bm == 128) spk_launch(k_dense<128, AA, AC>, grid, 256, 0, st, g);            \
        else if (bm == 64) spk_launch(k_dense<64, AA, AC>, grid, 128, 0, st, g);         \
        else spk_launch(k_dense<32, AA, AC>, grid, 64, 0, st, g);                        \
    } while (0)
    if (a_act == SPK_ACT_NONE) {
        if (act == SPK_ACT_NONE) LAUNCH_BM(0, 0); else if (act == SPK_ACT_SILU) LAUNCH_BM(0, 1); else LAUNCH_BM(0, 2);
    } else if (act == SPK_ACT_NONE) {
        if (a_act == SPK_ACT_SILU) LAUNCH_BM(1, 0); else if (a_act == SPK_ACT_SSP) LAUNCH_BM(2, 0); else LAUNCH_BM(3, 0);
    } else if (a_act == SPK_ACT_GIVEN) {
        if (act == SPK_ACT_SILU) LAUNCH_BM(3, 1); else LAUNCH_BM(3, 2);
    } else {   // both a backward prologue and a forward activation: rare, compiled for SiLU/ssp pairs of the same kind
        if (a_act == SPK_ACT_SILU && act == SPK_ACT_SILU) LAUNCH_BM(1, 1);
        else if (a_act == SPK_ACT_SSP && act == SPK_ACT_SSP) LAUNCH_BM(2, 2);
        else if (a_act == SPK_ACT_SILU) LAUNCH_BM(1, 2);
        else LAUNCH_BM(2, 1);
    }
#undef LAUNCH_BM
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

// Hopper tensor-core (wgmma), TMA and mbarrier primitives shared by the tensor-core kernels: thin inline-PTX wrappers and the
// one operand layout they all use -- K-major tiles of 16 floats (64 B rows) with the 64-byte swizzle.
//
// wgmma is issued by a whole warpgroup (4 warps, 128 threads) and leaves its fp32 accumulator in that warpgroup's registers.
// For a 64 x N accumulator (m64nNk8), thread t of the warpgroup holds element i of its fragment at
//     row = 16 * (t / 32) + (t % 32) / 4 + 8 * ((i / 2) % 2),    column = 8 * (i / 4) + 2 * (t % 4) + i % 2
// (wg_frag_row / wg_frag_col below).
#pragma once
#include "common.cuh"

constexpr int SPK_SW64_ROW = 64;               // bytes per operand row (16 floats)
constexpr int SPK_SW64_SBO = 8 * SPK_SW64_ROW; // 512 B between consecutive 8-row groups
constexpr int SPK_WG_ROWS_BYTES = 64 * SPK_SW64_ROW;   // 64 operand rows (one m64 slice) = 4096 B

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// one TMA bulk copy global -> shared, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// barrier over the 128 threads of one warpgroup (ids 1..15; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar(int id, int nthreads = 128) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// shared-memory matrix descriptor (sm_90), K-major, SWIZZLE_64B:
// start>>4 [0,14) | LBO (unused for swizzled K-major, 1) [16,30) | SBO>>4 [32,46) | layout 2 = 64B swizzle [62,64)
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(SPK_SW64_SBO >> 4) << 32) | (2ull << 62);
}
__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// byte offset of (row r, 16 B K-chunk c in 0..3) inside an operand tile: rows are 64 B, groups of 8 rows are 512 B atoms and
// the chunk index is XOR-swizzled with bits [1,3) of the row (Swizzle<2,4,3>, the pattern the tensor core applies to the
// byte address when the descriptor says SWIZZLE_64B).  Tiles are 512 B aligned.
__host__ __device__ __forceinline__ int tile_off(int r, int c) {
    return (r >> 3) * SPK_SW64_SBO + (r & 7) * SPK_SW64_ROW + ((c ^ ((r >> 1) & 3)) << 4);
}

// ---- wgmma -----------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// wait until at most N committed wgmma groups of the warpgroup are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ int wg_frag_row(int t, int i) { return 16 * ((t >> 5) & 3) + ((t & 31) >> 2) + 8 * ((i >> 1) & 1); }
__device__ __forceinline__ int wg_frag_col(int t, int i) { return 8 * (i >> 2) + 2 * (t & 3) + (i & 1); }

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, TF32 inputs, fp32 accumulate; scale_d == 0 overwrites D
#define SPK_WGMMA_PRE "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %"
__device__ __forceinline__ void wgmma_n8(float (&d)[4], uint64_t a, uint64_t b, int scale_d) {
    asm volatile(SPK_WGMMA_PRE "6, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0, %1, %2, %3}, %4, %5, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b, int scale_d) {
    asm volatile(SPK_WGMMA_PRE "18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, int scale_d) {
    asm volatile(SPK_WGMMA_PRE "34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(scale_d));
}
#undef SPK_WGMMA_PRE

// Issue the 3xTF32 products of one K-tile (16 floats = 2 k-steps) for one 64-column block on the calling warpgroup and
// commit them as ONE wgmma group, without waiting: its 64 rows of A (a_hi / a_lo: shared addresses of the warpgroup's
// first operand row) times 64 rows of W (b_hi / b_lo).  The tensor core truncates when it accumulates, which biases long
// K-sums toward zero; so the three products of the tile (small terms first: Al*Wh, Ah*Wl, then Ah*Wh) go into the FRESH
// accumulator t (the first product overwrites it), which the caller adds to its fp32 sum with round-to-nearest once the
// group has completed: the truncation never runs over more than one K-tile.
__device__ __forceinline__ void wg_ktile_3xtf32_issue(float (&t)[32], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                      uint32_t b_lo) {
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        wgmma_n64(t, make_desc(a_lo + 32 * ks), make_desc(b_hi + 32 * ks), ks);
        wgmma_n64(t, make_desc(a_hi + 32 * ks), make_desc(b_lo + 32 * ks), 1);
    }
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) wgmma_n64(t, make_desc(a_hi + 32 * ks), make_desc(b_hi + 32 * ks), 1);
    wgmma_commit();
}

// One K-tile for NB column blocks of 64 rows of W (b_hi / b_lo: tile start), each block issued, drained and added to
// acc[cb] in turn (wg_ktile_3xtf32_issue).
template <int NB>
__device__ __forceinline__ void wg_ktile_3xtf32(float (&acc)[NB][32], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi,
                                                uint32_t b_lo) {
#pragma unroll
    for (int cb = 0; cb < NB; ++cb) {
        float t[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) t[i] = 0.f;
        const uint32_t bo = (uint32_t)(cb * SPK_WG_ROWS_BYTES);
        wg_ktile_3xtf32_issue(t, a_hi, a_lo, b_hi + bo, b_lo + bo);
        wgmma_wait_all();
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[cb][i] += t[i];
    }
}

// Temperature replica exchange (parallel tempering) inside the captured device MD step (DESIGN.md section 25).
//
// The batch holds n_rungs * n_groups systems, rung-major: system k G + g is rung k of group g, and the systems of a group
// have the same atoms in the same order.  Attempt n tries the neighbouring pairs (k, k + 1) with k = n (mod 2) of every
// group (the deterministic even/odd scheme) and accepts one with the Metropolis test of Sugita and Okamoto; an accepted
// pair swaps the configurations of its two systems and rescales their momenta to the new temperatures.
//
// Two launches per attempt: k_remd_decide (one thread per pair) writes the decisions, the walker table and the
// statistics; k_remd_swap (one thread per atom and one per system) exchanges the rows of the decided pairs in every buffer
// of a by-value table and advances the attempt counter.  Pairs are disjoint and each row has one owner, so there are no
// atomics and the step is bitwise reproducible.  Both kernels return at once unless step[0] % every == 0.
#include "md_common.cuh"

namespace {

constexpr int DECIDE_T = 128;
constexpr int SWAP_T = 256;
// application index of the exchange draws: 2^63 + n, above every thermostat's counter and below the initializer's 2^64 - 1
constexpr uint64_t REMD_APPLICATION = 1ull << 63;

static_assert(SPK_REMD_MAX_BUFFERS == 16, "spk_remd_buffers_t holds 16 buffers");

__device__ __forceinline__ bool remd_gate(const int64_t* __restrict__ step, int64_t every) {
    return step == nullptr || (*step) % every == 0;
}

// pair i = g (K - 1) + k.  Delta = (1 / (kB T_k) - 1 / (kB T_k+1)) (U_k - U_k+1), U = energy * energy_conversion, all in
// fp64 with explicit roundings (no contraction), so a host restatement gets the same bits.
__global__ void __launch_bounds__(DECIDE_T) k_remd_decide(
    const float* __restrict__ energy, double energy_conversion, const double* __restrict__ temperature, double kB,
    int64_t n_groups, int K, uint64_t seed, const int64_t* __restrict__ step, int64_t every,
    const int64_t* __restrict__ attempt, int32_t* __restrict__ walker, int64_t* __restrict__ attempted,
    int64_t* __restrict__ accepted, uint8_t* __restrict__ decision) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_groups * (K - 1) || !remd_gate(step, every)) return;
    const int64_t n = attempt[0];
    const int64_t g = i / (K - 1);
    const int k = (int)(i - g * (K - 1));
    uint8_t swap = 0;
    if ((k & 1) == (int)(n & 1)) {
        const int64_t lo = (int64_t)k * n_groups + g, hi = lo + n_groups;
        const double b_lo = __ddiv_rn(1.0, __dmul_rn(kB, temperature[lo]));
        const double b_hi = __ddiv_rn(1.0, __dmul_rn(kB, temperature[hi]));
        const double u_lo = __dmul_rn((double)energy[lo], energy_conversion);
        const double u_hi = __dmul_rn((double)energy[hi], energy_conversion);
        const double delta = __dmul_rn(__dsub_rn(b_lo, b_hi), __dsub_rn(u_lo, u_hi));
        const uint4 x = philox_draw(seed, REMD_APPLICATION + (uint64_t)n, i);
        const double u = ((double)x.x + 0.5) * 2.3283064365386963e-10;
        swap = delta >= 0.0 || u < exp(delta);
        attempted[i] += 1;
        if (swap) {
            accepted[i] += 1;
            const int32_t w = walker[lo];
            walker[lo] = walker[hi];
            walker[hi] = w;
        }
    }
    decision[i] = swap;
}

__device__ __forceinline__ void swap_rows(float* __restrict__ d, int64_t w, int64_t a, int64_t b) {
    for (int64_t j = 0; j < w; ++j) {
        const float t = d[a * w + j];
        d[a * w + j] = d[b * w + j];
        d[b * w + j] = t;
    }
}

// item t < n_atoms: atom t; else system t - n_atoms.  The lower system of a swapping pair owns the exchange of its rows
// with the same rows of the system n_groups above it.
__global__ void __launch_bounds__(SWAP_T) k_remd_swap(
    const __grid_constant__ spk_remd_buffers_t b, float* __restrict__ momenta, const double* __restrict__ temperature,
    const int64_t* __restrict__ idx_m, const int32_t* __restrict__ sys_ptr, int64_t n_atoms, int64_t n_groups, int K,
    const uint8_t* __restrict__ decision, const int64_t* __restrict__ step, int64_t every, int64_t* __restrict__ attempt) {
    SPK_PDL_ENTER();
    if (!remd_gate(step, every)) return;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t == 0) attempt[0] += 1;               // k_remd_decide, which read it, has completed
    if (t >= n_atoms + n_groups * K) return;
    const bool atom = t < n_atoms;
    const int64_t s = atom ? idx_m[t] : t - n_atoms;
    const int64_t k = s / n_groups;
    if (k >= K - 1 || !decision[(s - k * n_groups) * (K - 1) + k]) return;
    const int64_t s2 = s + n_groups;
    const int64_t row = atom ? t : s, row2 = atom ? sys_ptr[s2] + (t - sys_ptr[s]) : s2;
    if (atom) {                                // p' = p sqrt(T_new / T_old), rounded once to fp32
        const double up = sqrt(temperature[s2] / temperature[s]), down = sqrt(temperature[s] / temperature[s2]);
        for (int d = 0; d < 3; ++d) {
            const double p_lo = (double)momenta[3 * row + d], p_hi = (double)momenta[3 * row2 + d];
            momenta[3 * row + d] = (float)(p_hi * down);
            momenta[3 * row2 + d] = (float)(p_lo * up);
        }
    }
    for (int i = 0; i < b.n_buffers; ++i)
        if ((b.per_atom[i] != 0) == atom) swap_rows(b.data[i], b.width[i], row, row2);
}

}  // namespace

extern "C" int spk_remd_exchange(const float* energy, double energy_conversion, const double* temperature, double kB,
                                 const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_groups,
                                 int32_t n_rungs, uint64_t seed, const int64_t* step, int64_t every, int64_t* attempt,
                                 int32_t* walker, int64_t* attempted, int64_t* accepted, uint8_t* decision,
                                 float* momenta, const spk_remd_buffers_t* buffers, spk_stream_t stream) {
    if (n_rungs < 2 || n_groups < 1 || n_atoms < 0 || every < 1 || !(kB > 0.0)) return SPK_ERR_ARG;
    if (n_groups > ((1ll << 31) - 1) / n_rungs || n_atoms + n_groups * n_rungs >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (!energy || !temperature || !attempt || !walker || !attempted || !accepted || !decision) return SPK_ERR_ARG;
    if (n_atoms > 0 && (!idx_m || !sys_ptr || !momenta)) return SPK_ERR_ARG;
    spk_remd_buffers_t b = {};
    if (buffers) b = *buffers;
    if (b.n_buffers < 0 || b.n_buffers > SPK_REMD_MAX_BUFFERS) return SPK_ERR_ARG;
    for (int i = 0; i < b.n_buffers; ++i) {
        if (!b.data[i] || b.width[i] < 1) return SPK_ERR_ARG;
        if (b.per_atom[i] && n_atoms == 0) return SPK_ERR_ARG;
    }
    cudaStream_t st = spk_st(stream);
    const int64_t n_pairs = n_groups * (n_rungs - 1);
    spk_launch(k_remd_decide, (unsigned)spk_cdiv(n_pairs, DECIDE_T), DECIDE_T, 0, st, energy, energy_conversion,
               temperature, kB, n_groups, (int)n_rungs, seed, step, every, (const int64_t*)attempt, walker, attempted,
               accepted, decision);
    spk_launch(k_remd_swap, (unsigned)spk_cdiv(n_atoms + n_groups * n_rungs, SWAP_T), SWAP_T, 0, st, b, momenta,
               temperature, idx_m, sys_ptr, n_atoms, n_groups, (int)n_rungs, (const uint8_t*)decision, step, every,
               attempt);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

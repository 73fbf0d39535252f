// Shared device/host helpers for the sm_90a (H100) kernels of the SchNetPack hot path.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/spk_b200.h"

#define SPK_CUDA_ERR(e) (-(1000 + (int)(e)))

#define SPK_LAUNCH_CHECK()                               \
    do {                                                 \
        cudaError_t _e = cudaGetLastError();             \
        if (_e != cudaSuccess) return SPK_CUDA_ERR(_e);  \
    } while (0)

static inline cudaStream_t spk_st(spk_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

// ---- programmatic dependent launch ----------------------------------------------------------------------------------
// One E+F evaluation is a chain of ~65 short kernels; a normal launch lets kernel n+1 start only after kernel n has drained
// and its completion has been processed.  Every kernel of the library is
// therefore launched with the programmatic-stream-serialization attribute and begins with
//     griddepcontrol.launch_dependents   -- the next kernel's CTAs may be scheduled as soon as all of ours are resident
//     griddepcontrol.wait                -- block until the previous kernel has completed and its writes are visible
// so the launch latency and CTA ramp-up of kernel n+1 overlap the tail of kernel n while the data dependence through
// global memory stays exactly that of a serial stream (the wait precedes every global access).  Works under stream capture (programmatic graph edges, CUDA >= 12.3).
#ifndef SPK_TIMELINE
#define SPK_TL_PHASE(kind) do { } while (0)
#define SPK_PDL_LAUNCH_DEPENDENTS() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define SPK_PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")
#else
// Debug build (-DSPK_TIMELINE): thread 0 of block 0 of EVERY kernel stamps
// %globaltimer at entry and when its griddepcontrol.wait returns (= the previous kernel has completed), tagged with the
// source line of the macro.  The differences between consecutive wait-return stamps are the kernels' durations INSIDE the
// programmatic-launch chain of a graph replay -- which neither CUDA events (they break the programmatic edges) nor ncu
// (serialised, cold) can show.  One buffer per translation unit (no relocatable device code), merged by time on the host.
static __device__ unsigned long long spk_tl_buf[2048];
static __device__ unsigned int spk_tl_n;
__device__ __forceinline__ void spk_tl_stamp(int line, int kind) {
    if ((blockIdx.x | blockIdx.y | blockIdx.z | threadIdx.x) == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        const unsigned int i = atomicAdd(&spk_tl_n, 1u);
        if (i < 1024) {
            spk_tl_buf[2 * i] = t;
            spk_tl_buf[2 * i + 1] = ((unsigned long long)line << 1) | (unsigned long long)kind;
        }
    }
}
// phase stamp inside a kernel (call from ONE lane; block 0 only records): kind >= 2, printed relative to the wait-return
__device__ __forceinline__ void spk_tl_phase(int kind) {
    if ((blockIdx.x | blockIdx.y | blockIdx.z) == 0) {
        unsigned long long t;
        asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
        const unsigned int i = atomicAdd(&spk_tl_n, 1u);
        if (i < 1024) {
            spk_tl_buf[2 * i] = t;
            spk_tl_buf[2 * i + 1] = (1ull << 40) | (unsigned long long)kind;
        }
    }
}
#define SPK_TL_PHASE(kind) spk_tl_phase(kind)
#define SPK_PDL_LAUNCH_DEPENDENTS()                                          \
    do {                                                                     \
        asm volatile("griddepcontrol.launch_dependents;" ::: "memory");      \
        spk_tl_stamp(__LINE__, 0);                                           \
    } while (0)
#define SPK_PDL_WAIT()                                                       \
    do {                                                                     \
        asm volatile("griddepcontrol.wait;" ::: "memory");                   \
        spk_tl_stamp(__LINE__, 1);                                           \
    } while (0)
#define SPK_TL_CAT2(a, b) a##b
#define SPK_TL_CAT(a, b) SPK_TL_CAT2(a, b)
// host: copy this translation unit's stamps out (n = number of stamps) and reset the counter
extern "C" int SPK_TL_CAT(spk_debug_timeline_, SPK_TU)(unsigned long long* host, unsigned int* n) {
    cudaDeviceSynchronize();
    unsigned int cnt = 0, zero = 0;
    cudaMemcpyFromSymbol(&cnt, spk_tl_n, sizeof(cnt));
    if (cnt > 1024) cnt = 1024;
    if (host && cnt) cudaMemcpyFromSymbol(host, spk_tl_buf, sizeof(unsigned long long) * 2 * cnt);
    cudaMemcpyToSymbol(spk_tl_n, &zero, sizeof(zero));
    *n = cnt;
    return 0;
}
#endif
#define SPK_PDL_ENTER()              \
    do {                             \
        SPK_PDL_LAUNCH_DEPENDENTS(); \
        SPK_PDL_WAIT();              \
    } while (0)

// Kernels that PACK static operands (weights in tensor-core operand layout) use SPK_PDL_WAIT_ONLY: they never trigger their
// dependents early, so every later kernel of the stream starts after the packed buffer is complete -- which lets the
// tensor-core kernels fetch those operands by TMA BEFORE their own griddepcontrol.wait (the copy then overlaps the previous
// kernel instead of sitting at the head of the critical path).
#define SPK_PDL_WAIT_ONLY() SPK_PDL_WAIT()

// compile with -DSPK_NO_PDL to restore plain launches (A/B builds); the library reads no environment variables
#ifdef SPK_NO_PDL
constexpr int SPK_PDL_ATTRS = 0;
#else
constexpr int SPK_PDL_ATTRS = 1;
#endif

template <typename... KArgs, typename... Args>
static inline void spk_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = SPK_PDL_ATTRS;
    (void)cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);   // errors surface in SPK_LAUNCH_CHECK()
}

static inline int64_t spk_cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

constexpr int SPK_NUM_SMS = 132;  // H100 SXM

// Per-device caches (a process may drive several GPUs): indexed by the CURRENT device of the calling thread, which the
// host side sets to the device of the tensors before every call.  Entries are write-once values, so concurrent callers
// at worst compute the same number twice.
constexpr int SPK_MAX_DEVICES = 64;
static inline int spk_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= SPK_MAX_DEVICES) dev = 0;
    return dev;
}

// SM count of the current device (132 on H100 SXM).
static inline int spk_num_sms() {
    static int n[SPK_MAX_DEVICES] = {0};
    const int dev = spk_device();
    if (!n[dev]) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0) v = SPK_NUM_SMS;
        n[dev] = v;
    }
    return n[dev];
}

// opt a kernel in to `bytes` of dynamic shared memory once per device (the attribute is per device and function)
struct SpkSmemOnce {
    unsigned char done[SPK_MAX_DEVICES] = {0};
    template <typename K>
    cudaError_t set(K kernel, int bytes) {
        const int dev = spk_device();
        if (done[dev]) return cudaSuccess;
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        if (e == cudaSuccess) done[dev] = 1;
        return e;
    }
};

__host__ __device__ __forceinline__ int spk_kp(int n_rbf) { return (n_rbf + 3) & ~3; }

// ---- activations (match torch fp32 semantics) --------------------------------------------------------------------
// silu(x) = x * sigmoid(x); torch: x / (1 + exp(-x))
__device__ __forceinline__ float spk_silu(float x) { return x / (1.0f + expf(-x)); }
__device__ __forceinline__ float spk_silu_grad(float x) {
    float s = 1.0f / (1.0f + expf(-x));
    return s * (1.0f + x * (1.0f - s));
}
// shifted softplus: softplus(x) - ln2, torch softplus threshold = 20 (nn/activations.py:22)
__device__ __forceinline__ float spk_ssp(float x) {
    float sp = (x > 20.0f) ? x : log1pf(expf(x));
    return sp - 0.6931471805599453f;
}
// The same function on the special-function unit for the fused SchNet block, which evaluates it 128 times per edge and is bound
// by those instructions: softplus(x) = max(x, 0) + log1p(t), t = exp(-|x|) in (0, 1]; exp and log through ex2.approx /
// lg2.approx (2^-22 relative / 2^-22.6 absolute), and log1p(t) = log(u) - ((u - 1) - t) / u with u = fl(1 + t) takes the
// rounding of 1 + t out again.  Absolute error ~1.2e-7 on values of order 0.1..1 (the libm version: ~6e-8).
__device__ __forceinline__ float spk_ssp_fast(float x) {
    float t;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-fabsf(x) * 1.4426950408889634f));
    const float u = 1.0f + t;
    const float l = __log2f(u) * 0.6931471805599453f - __fdividef((u - 1.0f) - t, u);
    return fmaxf(x, 0.0f) + l - 0.6931471805599453f;
}
__device__ __forceinline__ float spk_ssp_grad(float x) { return (x > 20.0f) ? 1.0f : 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ float spk_act(float x, int act) {
    if (act == SPK_ACT_SILU) return spk_silu(x);
    if (act == SPK_ACT_SSP) return spk_ssp(x);
    return x;
}
__device__ __forceinline__ float spk_act_grad(float x, int act) {
    if (act == SPK_ACT_SILU) return spk_silu_grad(x);
    if (act == SPK_ACT_SSP) return spk_ssp_grad(x);
    return 1.0f;
}

// activation value and derivative sharing one exp()
__device__ __forceinline__ void spk_act_both(float x, int act, float& y, float& dy) {
    if (act == SPK_ACT_SILU) {
        const float s = 1.0f / (1.0f + expf(-x));
        y = x * s;
        dy = s * (1.0f + x * (1.0f - s));
    } else if (act == SPK_ACT_SSP) {
        y = spk_ssp(x);
        dy = spk_ssp_grad(x);
    } else {
        y = x;
        dy = 1.0f;
    }
}

// (a * b + c) per component with IEEE round-to-nearest: on sm_90 scalar FFMA runs at the full fp32 rate, so the float2
// accumulators of the CUDA-core kernels are two independent FFMAs
__device__ __forceinline__ float2 spk_fma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

__device__ __forceinline__ float spk_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// first index r in [0, n] with ptr[r] >= target (ptr non-decreasing, length n+1)
__device__ __forceinline__ int spk_lower_bound(const int32_t* __restrict__ ptr, int n, int target) {
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (ptr[mid] < target) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// The same lower bound found by a whole warp: 32 probes per round instead of one, so the chain of DEPENDENT global loads is
// log32(n) + 1 long instead of log2(n) (5376 rows: 3 instead of 13 dependent L2 round trips at
// the head of every edge kernel).  All lanes must call; all get the result.
__device__ __forceinline__ int spk_lower_bound_warp(const int32_t* __restrict__ ptr, int n, int target) {
    const int lane = threadIdx.x & 31;
    int lo = 0, hi = n;                                        // the answer stays in [lo, hi]; ptr[n] is never read
    while (hi - lo > 32) {
        const long long span = hi - lo;
        const int p = lo + (int)(((lane + 1) * span) / 33);    // strictly increasing in lane, inside (lo, hi)
        const unsigned m = __ballot_sync(0xffffffffu, ptr[p] >= target);
        const int f = m ? __ffs(m) - 1 : 32;                   // first lane at or above the target
        const int new_hi = f == 32 ? hi : lo + (int)(((f + 1) * span) / 33);
        if (f > 0) lo = lo + (int)((f * span) / 33) + 1;       // lane f - 1 was still below it
        hi = new_hi;
    }
    const int p = lo + lane;
    const unsigned m = __ballot_sync(0xffffffffu, p < hi ? ptr[p] >= target : true);
    const int f = m ? __ffs(m) - 1 : 32;
    return min(lo + f, hi);
}
__device__ __forceinline__ int spk_block_row_begin_warp(const int32_t* __restrict__ ptr, int n, int n_edges, int nb, int b) {
    if (b <= 0) return 0;
    if (b >= nb) return n;
    return spk_lower_bound_warp(ptr, n, (int)(((long long)n_edges * b) / nb));
}

// Edge-balanced split of rows [0,n) over nb blocks: block b gets rows [row_begin(b), row_begin(b+1)).
__device__ __forceinline__ int spk_block_row_begin(const int32_t* __restrict__ ptr, int n, int n_edges, int nb, int b) {
    if (b <= 0) return 0;
    if (b >= nb) return n;
    long long target = ((long long)n_edges * b) / nb;
    // mix rows and edges so that edge-free rows are spread as well
    int r_e = spk_lower_bound(ptr, n, (int)target);
    return r_e;
}

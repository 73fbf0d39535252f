// Edge geometry, radial basis, cutoff, embedding and force assembly kernels (HBM-bound elementwise / segmented work).
// Reference: atomistic/distances.py:14-26, representation/painn.py:227-230, schnet.py:156-158, nn/radial.py,
// nn/cutoff.py:14-33, nn/activations.py:9-22, nn/scatter.py:26-34.
#include "segscan.cuh"

namespace {

constexpr float kPi = 3.14159265358979323846f;

// radial basis value and derivative for one (d, k)
__device__ __forceinline__ void rbf_eval(int kind, float d, float p0, float p1, float& v, float& dv) {
    if (kind == SPK_RBF_GAUSSIAN) {
        // nn/radial.py:11-15: coeff = -0.5 / w^2 ; exp(coeff * (d - mu)^2)
        float coeff = -0.5f / (p1 * p1);
        float diff = d - p0;
        v = expf(coeff * diff * diff);
        dv = 2.0f * coeff * diff * v;
    } else {
        // nn/radial.py:105-110: sin(f d) / d, d == 0 -> sin(f d) / 1
        float s, c;
        sincosf(p0 * d, &s, &c);
        if (d == 0.0f) {
            v = s;
            dv = p0 * c;
        } else {
            float inv = 1.0f / d;
            v = s * inv;
            dv = (p0 * c - v) * inv;
        }
    }
}

__device__ __forceinline__ void cutoff_eval(float d, float rc, float& fc, float& dfc) {
    // nn/cutoff.py:30-32: 0.5 (cos(d pi / rc) + 1) * (d < rc)
    float t = d * kPi / rc;
    float s, c;
    sincosf(t, &s, &c);
    bool in = d < rc;
    fc = in ? 0.5f * (c + 1.0f) : 0.0f;
    dfc = in ? (-0.5f * kPi / rc) * s : 0.0f;
}

__global__ void k_pairwise_fwd(const float* __restrict__ R, const int64_t* __restrict__ idx_i,
                               const int64_t* __restrict__ idx_j, const float* __restrict__ off, int64_t n_atoms,
                               int64_t n_edges, float* __restrict__ r_ij) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_edges * 3) return;
    int64_t e = t / 3;
    int c = (int)(t - e * 3);
    float o = off ? off[t] : 0.0f;
    const int64_t i = idx_i[e], j = idx_j[e];
    // out-of-range neighbour indices (the reference raises IndexError): never read out of bounds, poison the edge instead
    // (the graph build counts them in status[1] and empties the graph; the host raises on the first build of a new list)
    const bool ok = i >= 0 && i < n_atoms && j >= 0 && j < n_atoms;
    r_ij[t] = ok ? R[j * 3 + c] - R[i * 3 + c] + o : __int_as_float(0x7fc00000);
}

// one thread per (atom, component): deterministic sums over the receiver row and the sender row
__global__ void k_pairwise_bwd(const float* __restrict__ g, const int* __restrict__ rowptr,
                               const int* __restrict__ slot_eid, const int* __restrict__ sptr,
                               const int* __restrict__ pos_slot, int64_t n_atoms, float sign,
                               float* __restrict__ gR) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * 3) return;
    int64_t a = t / 3;
    int c = (int)(t - a * 3);
    float acc = 0.0f;
    for (int p = sptr[a]; p < sptr[a + 1]; ++p) acc += g[(int64_t)slot_eid[pos_slot[p]] * 3 + c];
    float sub = 0.0f;
    for (int s = rowptr[a]; s < rowptr[a + 1]; ++s) sub += g[(int64_t)slot_eid[s] * 3 + c];
    gR[t] = sign * (acc - sub);
}

// one thread per slot computes the geometry record, then KP threads-worth of radial values are produced by a loop
__global__ void k_edge_geometry(const float* __restrict__ r_ij, const int* __restrict__ slot_eid, int64_t n_edges,
                                int kind, int n_rbf, int KP, const float* __restrict__ p0, const float* __restrict__ p1,
                                float rc, const int* __restrict__ n_active, float* __restrict__ phi, float* __restrict__ dphi,
                                float* __restrict__ geo) {
    SPK_PDL_ENTER();
    // thread (s, c): slot s, 16-byte chunk c of its KP-float row -> float4 stores, consecutive threads write consecutive
    // chunks (a thread per scalar spent most of its instructions on 64-bit index arithmetic and re-deriving d)
    const int C = KP >> 2;
    const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_edges * C) return;
    const int s = (int)(t / C);
    if (n_active && s >= *n_active) return;      // CSR built from the active edges only: slots past its end do not exist
    const int c = (int)(t - (int64_t)s * C);
    const int64_t e = slot_eid ? (int64_t)slot_eid[s] : (int64_t)s;
    const float x = r_ij[e * 3 + 0], y = r_ij[e * 3 + 1], z = r_ij[e * 3 + 2];
    const float d = sqrtf(x * x + y * y + z * z);  // torch.norm(r_ij, dim=1)
    float v[4], dv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int k = c * 4 + u;
        v[u] = dv[u] = 0.0f;
        if (k < n_rbf) rbf_eval(kind, d, p0[k], p1 ? p1[k] : 0.0f, v[u], dv[u]);
    }
    reinterpret_cast<float4*>(phi)[t] = make_float4(v[0], v[1], v[2], v[3]);
    if (dphi) reinterpret_cast<float4*>(dphi)[t] = make_float4(dv[0], dv[1], dv[2], dv[3]);
    if (c == 0) {
        float fc, dfc;
        cutoff_eval(d, rc, fc, dfc);
        const float inv = 1.0f / d;  // d == 0 -> inf/NaN exactly like painn.py:228 (r_ij / d_ij)
        float4* gp = reinterpret_cast<float4*>(geo + (int64_t)s * SPK_GEO_STRIDE);
        gp[0] = make_float4(x * inv, y * inv, z * inv, d);
        gp[1] = make_float4(fc, dfc, inv, 0.0f);
    }
}

__global__ void k_rbf(const float* __restrict__ d, int64_t n, int kind, int n_rbf, const float* __restrict__ p0,
                      const float* __restrict__ p1, float* __restrict__ out, float* __restrict__ dout) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n * n_rbf) return;
    int64_t r = t / n_rbf;
    int k = (int)(t - r * n_rbf);
    float v, dv;
    rbf_eval(kind, d[r], p0[k], p1 ? p1[k] : 0.0f, v, dv);
    out[t] = v;
    if (dout) dout[t] = dv;
}

__global__ void k_cutoff(const float* __restrict__ d, int64_t n, float rc, float* __restrict__ out,
                         float* __restrict__ dout) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    float fc, dfc;
    cutoff_eval(d[t], rc, fc, dfc);
    out[t] = fc;
    if (dout) dout[t] = dfc;
}

__global__ void k_act(const float* __restrict__ x, int64_t n, int act, float* __restrict__ y, float* __restrict__ dy) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    float v = x[t];
    if (y) y[t] = spk_act(v, act);
    if (dy) dy[t] = spk_act_grad(v, act);
}

__global__ void k_embedding(const float* __restrict__ table, const int64_t* __restrict__ Z, int64_t n_atoms, int F4,
                            int n_rows, float* __restrict__ out) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * F4) return;
    int64_t a = t / F4;
    int c = (int)(t - a * F4);
    const int64_t z = Z[a];
    // nn.Embedding raises for z outside [0, n_rows); a kernel cannot raise, so the row is poisoned with NaN (loud in every
    // output) instead of being clamped to a valid element
    const float qn = __int_as_float(0x7fc00000);
    reinterpret_cast<float4*>(out)[t] = (z >= 0 && z < n_rows) ? reinterpret_cast<const float4*>(table)[z * F4 + c]
                                                                : make_float4(qn, qn, qn, qn);
}

// out[r, c] = sum_{s in row r} x[slot_eid[s], c]; thread per (r, c)
__global__ void k_segment_sum(const float* __restrict__ x, const int* __restrict__ rowptr,
                              const int* __restrict__ slot_eid, int64_t n_out, int C, float* __restrict__ out) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_out * C) return;
    int64_t r = t / C;
    int c = (int)(t - r * C);
    float acc = 0.0f;
    for (int s = rowptr[r]; s < rowptr[r + 1]; ++s) {
        int64_t e = slot_eid ? (int64_t)slot_eid[s] : (int64_t)s;
        acc += x[e * C + c];
    }
    out[t] = acc;
}

__global__ void k_add(const float* __restrict__ a, const float* __restrict__ b, int64_t n, float* __restrict__ out) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    out[t] = b ? a[t] + b[t] : a[t];
}

// velocity Verlet (md/integrators.py:59-70 half_step, :97-110 main_step) on the device-resident state: one thread per
// (atom, component).  forces arrive in MODEL units and are converted on the fly (md/calculators/base_calculator.py:96,
// force_conversion = energy_conversion / position_conversion); model_positions = positions * position_conversion is what the
// next force evaluation reads (base_calculator.py:_get_system_molecules).
__global__ void k_velocity_verlet(float* __restrict__ momenta, float* __restrict__ positions,
                                  float* __restrict__ model_positions, const float* __restrict__ forces,
                                  const float* __restrict__ masses, int64_t n_atoms, float dt, float f_conv, float p_conv,
                                  int drift) {
    SPK_PDL_ENTER();
    int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (t >= n_atoms * 3) return;
    const float p = fmaf(0.5f * dt, forces[t] * f_conv, momenta[t]);                 // p += 1/2 F dt
    momenta[t] = p;
    if (drift) {
        const float x = positions[t] + dt * p / masses[t / 3];                       // q += p / m dt
        positions[t] = x;
        if (model_positions) model_positions[t] = x * p_conv;
    }
}

// Per-system virial W_m[b][a] = sum_{e in m} g_e[b] r_e[a] (the strain derivative of atomistic/response.py:78-90 without the
// 1/V).  The edges of system m are the receiver slots [rowptr[sys_ptr[m]], rowptr[sys_ptr[m+1]]); CTAs take VIR_T
// consecutive slots and the two passes of segscan.cuh sum them in fp64 (seg_partials, then k_seg_finish), so the result is
// bitwise the same on every call for any mix of system sizes.  Padding pairs (distance 2 cutoff) have g_e = 0 and add
// nothing.
constexpr int VIR_T = 256;

__device__ __forceinline__ int64_t slot_of_sys(const int* __restrict__ rowptr, const int* __restrict__ sys_ptr, int64_t m) {
    return rowptr[sys_ptr[m]];
}

__global__ void __launch_bounds__(VIR_T) k_virial_partials(const float* __restrict__ g, const float* __restrict__ r,
                                                           const int* __restrict__ rowptr, const int* __restrict__ slot_eid,
                                                           const int* __restrict__ sys_ptr, int64_t n_sys,
                                                           double* __restrict__ sys_part, double* __restrict__ head) {
    SPK_PDL_ENTER();
    const int64_t s = (int64_t)blockIdx.x * VIR_T + threadIdx.x;
    const int64_t n_slots = slot_of_sys(rowptr, sys_ptr, n_sys);
    double v[9];
    int64_t m = 0, first = 0, end = 0;
#pragma unroll
    for (int c = 0; c < 9; ++c) v[c] = 0.0;
    if (s < n_slots) {
        int64_t lo = 0, hi = n_sys;   // last system whose first slot is <= s (skips empty systems)
        while (lo < hi) {
            const int64_t mid = (lo + hi + 1) >> 1;
            if (slot_of_sys(rowptr, sys_ptr, mid) <= s) lo = mid;
            else hi = mid - 1;
        }
        m = lo;
        const int64_t e = slot_eid[s];
        const double gx = g[3 * e], gy = g[3 * e + 1], gz = g[3 * e + 2];
        const double rx = r[3 * e], ry = r[3 * e + 1], rz = r[3 * e + 2];
        v[0] = gx * rx; v[1] = gx * ry; v[2] = gx * rz;
        v[3] = gy * rx; v[4] = gy * ry; v[5] = gy * rz;
        v[6] = gz * rx; v[7] = gz * ry; v[8] = gz * rz;
        first = slot_of_sys(rowptr, sys_ptr, m);
        end = slot_of_sys(rowptr, sys_ptr, m + 1);
    }
    seg_partials<VIR_T, 9>(v, n_slots, m, first, end, sys_part, head);
}

// Per-step model properties of DeviceMD (md/calculators/base_calculator.py:113-141): dst = src * conversion, and the
// device-side time series.  counter[0] = steps completed, counter[1] = records stored; both live in device memory and
// advance in stream order, so a captured step records at the right slot on every replay.  Step s (1-based) is recorded
// when s % every == 0.
__global__ void k_md_property(const float* __restrict__ src, int64_t n, float conversion, float* __restrict__ dst) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) dst[i] = src[i] * conversion;
}

__global__ void k_md_record(const float* __restrict__ src, int64_t n, const int64_t* __restrict__ counter, int64_t every,
                            int64_t capacity, float* __restrict__ buf) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t step = counter[0] + 1, slot = counter[1];
    if (i >= n || step % every != 0 || slot >= capacity) return;
    buf[slot * n + i] = src[i];
}

__global__ void k_md_record_velocities(const float* __restrict__ momenta, const float* __restrict__ masses, int64_t n,
                                       const int64_t* __restrict__ counter, int64_t every, int64_t capacity,
                                       float* __restrict__ buf) {
    SPK_PDL_ENTER();
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const int64_t step = counter[0] + 1, slot = counter[1];
    if (i >= 3 * n || step % every != 0 || slot >= capacity) return;
    buf[slot * 3 * n + i] = momenta[i] / masses[i / 3];
}

__global__ void k_md_record_advance(int64_t* __restrict__ counter, int64_t every, int64_t capacity) {
    SPK_PDL_ENTER();
    if (threadIdx.x != 0) return;
    const int64_t step = counter[0] + 1;
    counter[0] = step;
    if (step % every == 0 && counter[1] < capacity) counter[1] += 1;
}

}  // namespace

#define GRID1D(n, T) (unsigned)spk_cdiv((n), (T)), (T), 0, spk_st(stream)

extern "C" int spk_pairwise_fwd(const float* R, const int64_t* idx_i, const int64_t* idx_j, const float* offsets,
                                int64_t n_atoms, int64_t n_edges, float* r_ij, spk_stream_t stream) {
    if (n_edges < 0 || n_atoms < 0) return SPK_ERR_ARG;
    if (n_edges == 0) return SPK_OK;
    if (!R || !idx_i || !idx_j || !r_ij) return SPK_ERR_ARG;
    spk_launch(k_pairwise_fwd, GRID1D(n_edges * 3, 256), R, idx_i, idx_j, offsets, n_atoms, n_edges, r_ij);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_pairwise_bwd(const float* g_rij, const int32_t* rowptr, const int32_t* slot_eid, const int32_t* sptr,
                                const int32_t* pos_slot, int64_t n_atoms, float sign, float* g_R, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!rowptr || !sptr || !g_R) return SPK_ERR_ARG;
    spk_launch(k_pairwise_bwd, GRID1D(n_atoms * 3, 128), g_rij, rowptr, slot_eid, sptr, pos_slot, n_atoms, sign, g_R);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_edge_geometry(const float* r_ij, const int32_t* slot_eid, int64_t n_edges, int rbf_kind, int n_rbf,
                                 const float* rbf_p0, const float* rbf_p1, float cutoff, const int32_t* n_active,
                                 float* phi, float* dphi, float* geo, spk_stream_t stream) {
    // any n_rbf: the edge kernels that consume phi check their own limits (SO3net's convolution takes n_rbf > 32)
    if (n_edges < 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (rbf_kind != SPK_RBF_GAUSSIAN && rbf_kind != SPK_RBF_BESSEL) return SPK_ERR_ARG;
    if (n_edges == 0) return SPK_OK;
    if (!r_ij || !rbf_p0 || !phi || !geo) return SPK_ERR_ARG;
    if (rbf_kind == SPK_RBF_GAUSSIAN && !rbf_p1) return SPK_ERR_ARG;
    int KP = spk_kp(n_rbf);
    spk_launch(k_edge_geometry, GRID1D(n_edges * (KP / 4), 256), r_ij, slot_eid, n_edges, rbf_kind, n_rbf, KP, rbf_p0, rbf_p1,
                                                   cutoff, n_active, phi, dphi, geo);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_rbf_fwd(const float* d, int64_t n, int rbf_kind, int n_rbf, const float* rbf_p0,
                           const float* rbf_p1, float* out, float* dout, spk_stream_t stream) {
    if (n < 0 || n_rbf <= 0) return SPK_ERR_ARG;
    if (rbf_kind != SPK_RBF_GAUSSIAN && rbf_kind != SPK_RBF_BESSEL) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    if (!d || !rbf_p0 || !out || (rbf_kind == SPK_RBF_GAUSSIAN && !rbf_p1)) return SPK_ERR_ARG;
    spk_launch(k_rbf, GRID1D(n * n_rbf, 256), d, n, rbf_kind, n_rbf, rbf_p0, rbf_p1, out, dout);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_cosine_cutoff_fwd(const float* d, int64_t n, float cutoff, float* out, float* dout,
                                     spk_stream_t stream) {
    if (n < 0) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    if (!d || !out) return SPK_ERR_ARG;
    spk_launch(k_cutoff, GRID1D(n, 256), d, n, cutoff, out, dout);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_act_fwd(const float* x, int64_t n, int act, float* y, float* dy, spk_stream_t stream) {
    if (n < 0 || act < 0 || act > 2) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    if (!x) return SPK_ERR_ARG;
    spk_launch(k_act, GRID1D(n, 256), x, n, act, y, dy);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_embedding(const float* table, const int64_t* Z, int64_t n_atoms, int F, int n_rows, float* out,
                             spk_stream_t stream) {
    if (n_atoms < 0 || F <= 0 || (F & 3) || n_rows <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!table || !Z || !out) return SPK_ERR_ARG;
    spk_launch(k_embedding, GRID1D(n_atoms * (F / 4), 256), table, Z, n_atoms, F / 4, n_rows, out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_segment_sum(const float* x, const int32_t* rowptr, const int32_t* slot_eid, int64_t n_out, int C,
                               float* out, spk_stream_t stream) {
    if (n_out < 0 || C <= 0) return SPK_ERR_ARG;
    if (n_out == 0) return SPK_OK;
    if (!rowptr || !out) return SPK_ERR_ARG;
    spk_launch(k_segment_sum, GRID1D(n_out * C, 256), x, rowptr, slot_eid, n_out, C, out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_add(const float* a, const float* b, int64_t n, float* out, spk_stream_t stream) {
    if (n < 0) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    if (!a || !out) return SPK_ERR_ARG;
    spk_launch(k_add, GRID1D(n, 256), a, b, n, out);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_velocity_verlet(float* momenta, float* positions, float* model_positions, const float* forces,
                                      const float* masses, int64_t n_atoms, float dt, float force_conversion,
                                      float position_conversion, int drift, spk_stream_t stream) {
    if (n_atoms < 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!momenta || !forces || (drift && (!positions || !masses))) return SPK_ERR_ARG;
    spk_launch(k_velocity_verlet, GRID1D(n_atoms * 3, 256), momenta, positions, model_positions, forces, masses, n_atoms, dt,
               force_conversion, position_conversion, drift);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" size_t spk_pairwise_virial_workspace_bytes(int64_t n_edges, int64_t n_sys) {
    const int64_t nb = n_edges > 0 ? spk_cdiv(n_edges, VIR_T) : 0;
    return sizeof(double) * 9 * (size_t)((n_sys > 0 ? n_sys : 0) + nb + 1);
}

extern "C" int spk_pairwise_virial(const float* g_rij, const float* r_ij, const int32_t* rowptr, const int32_t* slot_eid,
                                   const int32_t* sys_ptr, int64_t n_edges, int64_t n_sys, double* virial, void* workspace,
                                   size_t workspace_bytes, spk_stream_t stream) {
    if (n_edges < 0 || n_sys <= 0 || n_edges >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (!rowptr || !sys_ptr || !virial || !workspace) return SPK_ERR_ARG;
    if (workspace_bytes < spk_pairwise_virial_workspace_bytes(n_edges, n_sys)) return SPK_ERR_ARG;
    if (n_edges > 0 && (!g_rij || !r_ij || !slot_eid)) return SPK_ERR_ARG;
    double* sys_part = reinterpret_cast<double*>(workspace);
    double* head = sys_part + 9 * n_sys;
    if (n_edges > 0)
        spk_launch(k_virial_partials, (unsigned)spk_cdiv(n_edges, VIR_T), VIR_T, 0, spk_st(stream), g_rij, r_ij, rowptr,
                   slot_eid, sys_ptr, n_sys, sys_part, head);
    spk_launch(k_seg_finish<VIR_T, 9>, (unsigned)n_sys, SEG_FIN_T, 0, spk_st(stream), rowptr, sys_ptr, sys_part, head,
               virial);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

namespace {
// the per-system pass of k_seg_finish<VIR_T, 9> that adds the totals to virial (after the reciprocal Ewald virial)
__global__ void __launch_bounds__(SEG_FIN_T) k_virial_finish_add(const int32_t* __restrict__ rowptr,
                                                                 const int32_t* __restrict__ sys_ptr,
                                                                 const double* __restrict__ sys_part,
                                                                 const double* __restrict__ head, double* __restrict__ out) {
    __shared__ double red[9][SEG_FIN_T];
    SPK_PDL_ENTER();
    const int64_t s = blockIdx.x;
    seg_finish_block<VIR_T, 9>(rowptr, sys_ptr, sys_part, head, s, red);
    if (threadIdx.x < 9) out[s * 9 + threadIdx.x] += red[threadIdx.x][0];
}
}  // namespace

extern "C" int spk_pairwise_virial_add(const float* g_rij, const float* r_ij, const int32_t* rowptr,
                                       const int32_t* slot_eid, const int32_t* sys_ptr, int64_t n_edges, int64_t n_sys,
                                       double* virial, void* workspace, size_t workspace_bytes, spk_stream_t stream) {
    if (n_edges < 0 || n_sys <= 0 || n_edges >= (1ll << 31) - 1) return SPK_ERR_ARG;
    if (!rowptr || !sys_ptr || !virial || !workspace) return SPK_ERR_ARG;
    if (workspace_bytes < spk_pairwise_virial_workspace_bytes(n_edges, n_sys)) return SPK_ERR_ARG;
    if (n_edges > 0 && (!g_rij || !r_ij || !slot_eid)) return SPK_ERR_ARG;
    double* sys_part = reinterpret_cast<double*>(workspace);
    double* head = sys_part + 9 * n_sys;
    if (n_edges > 0)
        spk_launch(k_virial_partials, (unsigned)spk_cdiv(n_edges, VIR_T), VIR_T, 0, spk_st(stream), g_rij, r_ij, rowptr,
                   slot_eid, sys_ptr, n_sys, sys_part, head);
    spk_launch(k_virial_finish_add, (unsigned)n_sys, SEG_FIN_T, 0, spk_st(stream), rowptr, sys_ptr, sys_part, head,
               virial);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_property(const float* src, int64_t n, float conversion, float* dst, spk_stream_t stream) {
    if (n < 0) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    if (!src || !dst) return SPK_ERR_ARG;
    spk_launch(k_md_property, GRID1D(n, 256), src, n, conversion, dst);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_record(const float* src, int64_t n, const int64_t* counter, int64_t every, int64_t capacity,
                             float* buf, spk_stream_t stream) {
    if (n < 0 || every <= 0 || capacity <= 0) return SPK_ERR_ARG;
    if (n == 0) return SPK_OK;
    if (!src || !counter || !buf) return SPK_ERR_ARG;
    spk_launch(k_md_record, GRID1D(n, 256), src, n, counter, every, capacity, buf);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_record_advance(int64_t* counter, int64_t every, int64_t capacity, spk_stream_t stream) {
    if (!counter || every <= 0 || capacity <= 0) return SPK_ERR_ARG;
    spk_launch(k_md_record_advance, 1, 32, 0, spk_st(stream), counter, every, capacity);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

extern "C" int spk_md_record_velocities(const float* momenta, const float* masses, int64_t n_atoms,
                                        const int64_t* counter, int64_t every, int64_t capacity, float* buf,
                                        spk_stream_t stream) {
    if (n_atoms < 0 || every <= 0 || capacity <= 0) return SPK_ERR_ARG;
    if (n_atoms == 0) return SPK_OK;
    if (!momenta || !masses || !counter || !buf) return SPK_ERR_ARG;
    spk_launch(k_md_record_velocities, GRID1D(3 * n_atoms, 256), momenta, masses, n_atoms, counter, every, capacity, buf);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

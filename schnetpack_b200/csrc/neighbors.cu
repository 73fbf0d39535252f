// Device-resident neighbour list (SURVEY.md section 8, "next" row f1): a linked-cell search per system of a collated
// batch, replacing the CPU round trip of the reference (md/neighborlist_md.py:129,213-232 copies Z/R/cell to the host and
// calls matscipy/ASE every rebuild).  Contract = transform/neighborlist.py:428-553 (TorchNeighborList; the ASE / matscipy /
// vesin front ends :213-286 return the same set):
//   pair (i, j, S) listed  <=>  | R[j] - R[i] + S @ cell | < cutoff,  S integer, S_a = 0 on non-periodic axes,
//   (i == j, S == 0) excluded, self images (i == j, S != 0) listed;  offsets = S @ cell;  sorted by idx_i.
// Positions may lie any number of cells away from the cell, and the rows of non-periodic axes may be zero.
// Everything is enqueue-only on the caller's stream (no host synchronisation: the pair count stays on the device and the
// tail of the fixed-capacity output can be padded with edges that lie outside the cutoff), deterministic (no atomics: the
// atoms are ordered by cell with a stable radix sort, rows are written in traversal order), and works in fp32 with the
// same expression the model uses for r_ij (R[j] - R[i] + offsets), so every listed pair is inside the cutoff as the
// model sees it.
//
// Grid: per system, n_a = floor(height_a / cutoff) cells along each periodic axis (height = distance between the cell
// faces), 1 on non-periodic axes, coarsened until the system has at most one cell per atom; the search visits `reach`
// cells on each side (1, or ceil(cutoff / height) images when the cell is thinner than the cutoff), image shifts included.
#include <cub/cub.cuh>

#include "cell_grid.cuh"

namespace {

// One warp per atom.  FILL == false: count the neighbours of atom i; FILL == true: write them at row_start[i].
template <bool FILL>
__global__ void __launch_bounds__(256) k_nl_search(const float* __restrict__ R, const int32_t* __restrict__ sys_ptr,
                                                   int n_sys, int n_atoms, const SysGrid* __restrict__ grid,
                                                   const int* __restrict__ cell_of, const int* __restrict__ wrap,
                                                   const int* __restrict__ sorted_atom, const int* __restrict__ cell_start,
                                                   const int* __restrict__ cell_end, float cutoff2,
                                                   int* __restrict__ deg, const int* __restrict__ row_start,
                                                   long long capacity, int pad, float cutoff,
                                                   int64_t* __restrict__ idx_i, int64_t* __restrict__ idx_j,
                                                   float* __restrict__ offsets, int32_t* __restrict__ shifts) {
    SPK_PDL_ENTER();
    const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n_atoms) return;
    const int s = find_system(sys_ptr, n_sys, i);
    const SysGrid& g = grid[s];
    const float xi = R[i * 3 + 0], yi = R[i * 3 + 1], zi = R[i * 3 + 2];
    const int wi0 = wrap[i * 3 + 0], wi1 = wrap[i * 3 + 1], wi2 = wrap[i * 3 + 2];
    int lc = cell_of[i] - g.cell_base;
    const int c2 = lc % g.n[2];
    lc /= g.n[2];
    const int c1 = lc % g.n[1], c0 = lc / g.n[1];
    // padding (fixed-capacity mode): the unused capacity P is spread over the rows -- row i is followed by
    // floor((i+1) P / N) - floor(i P / N) inert self pairs -- so idx_i stays sorted and no atom collects a long row
    long long out = 0, pads_before = 0, pads_mine = 0;
    if (FILL) {
        const long long total = row_start[n_atoms];
        const long long P = (pad && capacity > total) ? capacity - total : 0;
        pads_before = ((long long)i * P) / n_atoms;
        pads_mine = ((long long)(i + 1) * P) / n_atoms - pads_before;
        out = (long long)row_start[i] + pads_before;
    }
    int count = 0;
    for (int d0 = -g.reach[0]; d0 <= g.reach[0]; ++d0) {
        const int t0 = c0 + d0;
        const int s0 = (t0 >= 0 ? t0 / g.n[0] : -((-t0 + g.n[0] - 1) / g.n[0]));      // floor division: image of the cell
        const int n0 = t0 - s0 * g.n[0];
        for (int d1 = -g.reach[1]; d1 <= g.reach[1]; ++d1) {
            const int t1 = c1 + d1;
            const int s1 = (t1 >= 0 ? t1 / g.n[1] : -((-t1 + g.n[1] - 1) / g.n[1]));
            const int n1 = t1 - s1 * g.n[1];
            for (int d2 = -g.reach[2]; d2 <= g.reach[2]; ++d2) {
                const int t2 = c2 + d2;
                const int s2 = (t2 >= 0 ? t2 / g.n[2] : -((-t2 + g.n[2] - 1) / g.n[2]));
                const int n2 = t2 - s2 * g.n[2];
                const int cj = g.cell_base + (n0 * g.n[1] + n1) * g.n[2] + n2;
                const int beg = cell_start[cj], end = cell_end[cj];
                for (int p0 = beg; p0 < end; p0 += 32) {
                    const int p = p0 + lane;
                    bool hit = false;
                    int j = 0, S0 = 0, S1 = 0, S2 = 0;
                    float ox = 0.f, oy = 0.f, oz = 0.f;
                    if (p < end) {
                        j = sorted_atom[p];
                        // image vector relative to the UNWRAPPED input positions
                        S0 = s0 + wi0 - wrap[j * 3 + 0];
                        S1 = s1 + wi1 - wrap[j * 3 + 1];
                        S2 = s2 + wi2 - wrap[j * 3 + 2];
                        if (!(j == i && S0 == 0 && S1 == 0 && S2 == 0)) {
                            ox = (float)S0 * g.c[0] + (float)S1 * g.c[3] + (float)S2 * g.c[6];     // offsets = S @ cell
                            oy = (float)S0 * g.c[1] + (float)S1 * g.c[4] + (float)S2 * g.c[7];
                            oz = (float)S0 * g.c[2] + (float)S1 * g.c[5] + (float)S2 * g.c[8];
                            const float dx = R[j * 3 + 0] - xi + ox, dy = R[j * 3 + 1] - yi + oy, dz = R[j * 3 + 2] - zi + oz;
                            hit = dx * dx + dy * dy + dz * dz < cutoff2;
                        }
                    }
                    const unsigned m = __ballot_sync(0xffffffffu, hit);
                    if (FILL) {
                        if (hit) {
                            const long long e = out + __popc(m & ((1u << lane) - 1u));
                            if (e < capacity) {
                                idx_i[e] = i;
                                idx_j[e] = j;
                                offsets[e * 3 + 0] = ox;
                                offsets[e * 3 + 1] = oy;
                                offsets[e * 3 + 2] = oz;
                                if (shifts) {
                                    shifts[e * 3 + 0] = S0;
                                    shifts[e * 3 + 1] = S1;
                                    shifts[e * 3 + 2] = S2;
                                }
                            }
                        }
                        out += __popc(m);
                    } else {
                        count += __popc(m);
                    }
                }
            }
        }
    }
    if (!FILL && lane == 0) deg[i] = count;
    if (FILL) {
        for (long long t = lane; t < pads_mine; t += 32) {
            const long long e = out + t;
            if (e >= capacity) break;
            idx_i[e] = i;                        // self pair at distance 2 cutoff: the cosine cutoff and its derivative vanish,
            idx_j[e] = i;                        // so it contributes nothing to energies or forces
            offsets[e * 3 + 0] = 2.0f * cutoff;
            offsets[e * 3 + 1] = 0.f;
            offsets[e * 3 + 2] = 0.f;
            if (shifts) shifts[e * 3 + 0] = shifts[e * 3 + 1] = shifts[e * 3 + 2] = 0;
        }
    }
}

// n_pairs[0] = pairs found, n_pairs[1] = 1 if they did not fit
__global__ void k_nl_finish(const int* __restrict__ row_start, int n_atoms, long long capacity,
                            int64_t* __restrict__ n_pairs) {
    SPK_PDL_ENTER();
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        const long long total = row_start[n_atoms];
        n_pairs[0] = total;
        n_pairs[1] = total > capacity ? 1 : 0;
    }
}

struct NlLayout {
    size_t grid, total, cell_of, atom_id, sorted_cell, sorted_atom, wrap, cell_start, cell_end, deg, row_start, cub, end;
    size_t cub_bytes;
};

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

NlLayout nl_layout(int64_t n_atoms, int64_t n_sys) {
    NlLayout L;
    size_t o = 0;
    const size_t ncell = (size_t)(n_atoms + n_sys + 1);
    L.grid = o; o = align256(o + sizeof(SysGrid) * (size_t)(n_sys > 0 ? n_sys : 1));
    L.total = o; o = align256(o + 16);
    L.cell_of = o; o = align256(o + 4 * (size_t)n_atoms);
    L.atom_id = o; o = align256(o + 4 * (size_t)n_atoms);
    L.sorted_cell = o; o = align256(o + 4 * (size_t)n_atoms);
    L.sorted_atom = o; o = align256(o + 4 * (size_t)n_atoms);
    L.wrap = o; o = align256(o + 12 * (size_t)n_atoms);
    L.cell_start = o; o = align256(o + 4 * ncell);
    L.cell_end = o; o = align256(o + 4 * ncell);
    L.deg = o; o = align256(o + 4 * (size_t)(n_atoms + 1));
    L.row_start = o; o = align256(o + 4 * (size_t)(n_atoms + 1));
    size_t sort_b = 0, scan_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr,
                                    (int)n_atoms);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int*)nullptr, (int*)nullptr, (int)(n_atoms + 1));
    L.cub_bytes = sort_b > scan_b ? sort_b : scan_b;
    L.cub = o; o = align256(o + L.cub_bytes);
    L.end = o;
    return L;
}

}  // namespace

extern "C" size_t spk_neighbor_list_workspace_bytes(int64_t n_atoms, int64_t n_sys) {
    if (n_atoms < 0 || n_sys < 0) return 0;
    return nl_layout(n_atoms, n_sys).end;
}

extern "C" int spk_neighbor_list(const float* R, const float* cell, const uint8_t* pbc, const int32_t* sys_ptr,
                                 int64_t n_atoms, int64_t n_sys, float cutoff, int64_t capacity, int pad, int64_t* idx_i,
                                 int64_t* idx_j, float* offsets, int32_t* shifts, int64_t* n_pairs, void* workspace,
                                 size_t workspace_bytes, spk_stream_t stream) {
    if (n_atoms < 0 || n_sys < 0 || capacity < 0 || !(cutoff > 0.f)) return SPK_ERR_ARG;
    if (n_atoms > 0x3fffffff) return SPK_ERR_UNSUPPORTED;
    if (!n_pairs) return SPK_ERR_ARG;
    cudaStream_t st = spk_st(stream);
    if (n_atoms == 0 || n_sys == 0) {
        cudaError_t e = cudaMemsetAsync(n_pairs, 0, 16, st);
        return e == cudaSuccess ? SPK_OK : SPK_CUDA_ERR(e);
    }
    if (!R || !cell || !pbc || !sys_ptr || !workspace) return SPK_ERR_ARG;
    if (capacity > 0 && (!idx_i || !idx_j || !offsets)) return SPK_ERR_ARG;
    const NlLayout L = nl_layout(n_atoms, n_sys);
    if (workspace_bytes < L.end) return SPK_ERR_ARG;
    uint8_t* ws = static_cast<uint8_t*>(workspace);
    SysGrid* grid = reinterpret_cast<SysGrid*>(ws + L.grid);
    int* total = reinterpret_cast<int*>(ws + L.total);
    int* cell_of = reinterpret_cast<int*>(ws + L.cell_of);
    int* atom_id = reinterpret_cast<int*>(ws + L.atom_id);
    int* sorted_cell = reinterpret_cast<int*>(ws + L.sorted_cell);
    int* sorted_atom = reinterpret_cast<int*>(ws + L.sorted_atom);
    int* wrap = reinterpret_cast<int*>(ws + L.wrap);
    int* cell_start = reinterpret_cast<int*>(ws + L.cell_start);
    int* cell_end = reinterpret_cast<int*>(ws + L.cell_end);
    int* deg = reinterpret_cast<int*>(ws + L.deg);
    int* row_start = reinterpret_cast<int*>(ws + L.row_start);
    const int N = (int)n_atoms, B = (int)n_sys;
    cudaError_t e = cudaMemsetAsync(ws + L.cell_start, 0, L.deg - L.cell_start, st);      // empty cells: start == end == 0
    if (e == cudaSuccess) e = cudaMemsetAsync(deg, 0, 4 * (size_t)(N + 1), st);
    if (e != cudaSuccess) return SPK_CUDA_ERR(e);
    spk_launch(k_nl_setup, 1, 1024, 0, st, cell, pbc, sys_ptr, B, cutoff, grid, total,
               (const int*)nullptr);
    spk_launch(k_nl_bin, (unsigned)spk_cdiv(N, 256), 256, 0, st, R, sys_ptr, B, N, (const SysGrid*)grid, cell_of, atom_id, wrap,
               (const int*)nullptr);
    size_t cub_bytes = L.cub_bytes;
    e = cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, (const int*)cell_of, sorted_cell, (const int*)atom_id,
                                        sorted_atom, N, 0, 32, st);
    if (e != cudaSuccess) return SPK_CUDA_ERR(e);
    spk_launch(k_nl_cell_bounds, (unsigned)spk_cdiv(N, 256), 256, 0, st, (const int*)sorted_cell, N, cell_start, cell_end,
               (const int*)nullptr);
    const unsigned gw = (unsigned)spk_cdiv((int64_t)N * 32, 256);
    spk_launch(k_nl_search<false>, gw, 256, 0, st, R, sys_ptr, B, N, (const SysGrid*)grid, (const int*)cell_of,
               (const int*)wrap, (const int*)sorted_atom, (const int*)cell_start, (const int*)cell_end, cutoff * cutoff, deg,
               (const int*)row_start, (long long)capacity, 0, cutoff, idx_i, idx_j, offsets, shifts);
    cub_bytes = L.cub_bytes;
    e = cub::DeviceScan::ExclusiveSum(ws + L.cub, cub_bytes, (const int*)deg, row_start, N + 1, st);
    if (e != cudaSuccess) return SPK_CUDA_ERR(e);
    if (capacity > 0)
        spk_launch(k_nl_search<true>, gw, 256, 0, st, R, sys_ptr, B, N, (const SysGrid*)grid, (const int*)cell_of,
                   (const int*)wrap, (const int*)sorted_atom, (const int*)cell_start, (const int*)cell_end, cutoff * cutoff,
                   deg, (const int*)row_start, (long long)capacity, pad, cutoff, idx_i, idx_j, offsets, shifts);
    spk_launch(k_nl_finish, 1, 32, 0, st, (const int*)row_start, N, (long long)capacity, n_pairs);
    SPK_LAUNCH_CHECK();
    return SPK_OK;
}

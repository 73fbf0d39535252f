// The cell grid of the device neighbour list (neighbors.cu), shared with every search that walks the same cells: the
// radial distribution function of structure.cu bins the pairs the neighbour list would list, at its own cutoff, without
// writing them out.  Per system, n_a = floor(height_a / cutoff) cells along each periodic axis (height = distance between
// the cell faces), 1 on non-periodic axes, coarsened until the system has at most one cell per atom; a search visits
// `reach` cells on each side (1, or ceil(cutoff / height) images when the cell is thinner than the cutoff).
//
// gate (nullable) is a device flag: with it, the kernels return at once when gate[0] == 0, so a hook inside a captured step
// builds the grid only on the steps it samples.
#pragma once
#include "common.cuh"

namespace {

__device__ __forceinline__ bool grid_gated_off(const int* gate) { return gate != nullptr && *gate == 0; }

struct SysGrid {
    float c[9];        // cell rows a, b, c
    float inv[9];      // inverse(cell): frac = R @ inv
    int n[3];          // cells per axis
    int reach[3];      // neighbour cells visited on each side
    int pbc[3];
    int cell_base;     // first global cell id of this system
    int any_pbc;
};

__device__ __forceinline__ int find_system(const int32_t* __restrict__ sys_ptr, int n_sys, int atom) {
    int lo = 0, hi = n_sys;                      // largest s with sys_ptr[s] <= atom
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (sys_ptr[mid] <= atom) lo = mid; else hi = mid;
    }
    return lo;
}

// unit vector along x cross y
__device__ void cross_unit(const double* x, const double* y, double* out) {
    const double z[3] = {x[1] * y[2] - x[2] * y[1], x[2] * y[0] - x[0] * y[2], x[0] * y[1] - x[1] * y[0]};
    const double il = 1.0 / sqrt(z[0] * z[0] + z[1] * z[1] + z[2] * z[2]);
    for (int k = 0; k < 3; ++k) out[k] = z[k] * il;
}

// The cell with the rows of the non-periodic axes replaced by an orthonormal completion of the periodic rows: the unit
// normal of two periodic rows, or two orthogonal unit vectors normal to one.  Fractional coordinates, heights and wraps
// along the periodic axes then depend on the periodic rows only, and a sheet or a wire whose non-periodic rows are zero
// (ase.build.graphene(vacuum=None), nanotubes) gets an invertible cell; offsets still use the caller's rows, whose
// images are 0 on those axes.  A degenerate PERIODIC row is invalid input and is not detected here.
__device__ void complete_cell(const float* c, const int* pbc, double* m) {
    int per[3], non[3], n_per = 0, n_non = 0;
    for (int a = 0; a < 3; ++a) {
        for (int k = 0; k < 3; ++k) m[3 * a + k] = c[3 * a + k];
        if (pbc[a]) per[n_per++] = a; else non[n_non++] = a;
    }
    if (n_per == 2) {
        cross_unit(m + 3 * per[0], m + 3 * per[1], m + 3 * non[0]);
    } else if (n_per == 1) {
        const double* p = m + 3 * per[0];
        int least = 0;                                               // the coordinate axis least aligned with p
        for (int k = 1; k < 3; ++k)
            if (fabs(p[k]) < fabs(p[least])) least = k;
        double e[3] = {0.0, 0.0, 0.0};
        e[least] = 1.0;
        cross_unit(p, e, m + 3 * non[0]);
        cross_unit(p, m + 3 * non[0], m + 3 * non[1]);
    }
}

__global__ void __launch_bounds__(1024) k_nl_setup(const float* __restrict__ cell, const uint8_t* __restrict__ pbc,
                                                   const int32_t* __restrict__ sys_ptr, int n_sys, float cutoff,
                                                   SysGrid* __restrict__ grid, int* __restrict__ total_cells,
                                                   const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (grid_gated_off(gate)) return;
    const float rc = cutoff * 1.0001f;           // cells a hair wider than the cutoff: binning is done in fp32
    for (int s = threadIdx.x; s < n_sys; s += blockDim.x) {
        SysGrid g;
        bool any = false;
        for (int a = 0; a < 3; ++a) {
            g.pbc[a] = pbc[s * 3 + a] ? 1 : 0;
            any |= g.pbc[a] != 0;
        }
        for (int k = 0; k < 9; ++k) g.c[k] = cell[s * 9 + k];
        g.any_pbc = any ? 1 : 0;
        for (int a = 0; a < 3; ++a) {
            g.n[a] = 1;
            g.reach[a] = 0;
        }
        for (int k = 0; k < 9; ++k) g.inv[k] = 0.f;
        if (any) {
            // inverse of the completed cell by cofactors in double (3x3)
            double m[9];
            complete_cell(g.c, g.pbc, m);
            const double a0 = m[0], a1 = m[1], a2 = m[2], b0 = m[3], b1 = m[4], b2 = m[5], c0 = m[6], c1 = m[7], c2 = m[8];
            const double det = a0 * (b1 * c2 - b2 * c1) - a1 * (b0 * c2 - b2 * c0) + a2 * (b0 * c1 - b1 * c0);
            const double id = 1.0 / det;
            double inv[9];
            inv[0] = (b1 * c2 - b2 * c1) * id; inv[1] = (a2 * c1 - a1 * c2) * id; inv[2] = (a1 * b2 - a2 * b1) * id;
            inv[3] = (b2 * c0 - b0 * c2) * id; inv[4] = (a0 * c2 - a2 * c0) * id; inv[5] = (a2 * b0 - a0 * b2) * id;
            inv[6] = (b0 * c1 - b1 * c0) * id; inv[7] = (a1 * c0 - a0 * c1) * id; inv[8] = (a0 * b1 - a1 * b0) * id;
            for (int k = 0; k < 9; ++k) g.inv[k] = (float)inv[k];
            const int na = sys_ptr[s + 1] - sys_ptr[s];
            for (int a = 0; a < 3; ++a) {
                if (!g.pbc[a]) continue;
                // height_a = 1 / |column a of inverse(cell)|  (neighborlist.py:529-531)
                const double il = sqrt(inv[a] * inv[a] + inv[3 + a] * inv[3 + a] + inv[6 + a] * inv[6 + a]);
                const double h = 1.0 / il;
                int n = (int)floor(h / rc);
                if (n < 1) n = 1;
                g.n[a] = n;
                g.reach[a] = (int)ceil(rc / (h / n));
            }
            while ((long long)g.n[0] * g.n[1] * g.n[2] > (long long)(na > 1 ? na : 1)) {   // at most one cell per atom
                int big = 0;
                if (g.n[1] > g.n[big]) big = 1;
                if (g.n[2] > g.n[big]) big = 2;
                if (g.n[big] <= 1) break;
                g.n[big] -= 1;
            }
        }
        grid[s] = g;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int base = 0;
        for (int s = 0; s < n_sys; ++s) {
            grid[s].cell_base = base;
            base += grid[s].n[0] * grid[s].n[1] * grid[s].n[2];
        }
        *total_cells = base;
    }
}

// cell id and periodic wrap of every atom
__global__ void k_nl_bin(const float* __restrict__ R, const int32_t* __restrict__ sys_ptr, int n_sys, int n_atoms,
                         const SysGrid* __restrict__ grid, int* __restrict__ cell_of, int* __restrict__ atom_id,
                         int* __restrict__ wrap, const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (grid_gated_off(gate)) return;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_atoms) return;
    const int s = find_system(sys_ptr, n_sys, i);
    const SysGrid& g = grid[s];
    int w[3] = {0, 0, 0}, ci[3] = {0, 0, 0};
    if (g.any_pbc) {
        const float x = R[i * 3 + 0], y = R[i * 3 + 1], z = R[i * 3 + 2];
        for (int a = 0; a < 3; ++a) {
            if (!g.pbc[a]) continue;
            const float f = x * g.inv[a] + y * g.inv[3 + a] + z * g.inv[6 + a];
            const float fl = floorf(f);
            w[a] = (int)fl;
            int cc = (int)((f - fl) * (float)g.n[a]);
            ci[a] = cc < 0 ? 0 : (cc >= g.n[a] ? g.n[a] - 1 : cc);
        }
    }
    cell_of[i] = g.cell_base + (ci[0] * g.n[1] + ci[1]) * g.n[2] + ci[2];
    atom_id[i] = i;
    wrap[i * 3 + 0] = w[0];
    wrap[i * 3 + 1] = w[1];
    wrap[i * 3 + 2] = w[2];
}

// boundaries of the cell segments in the cell-sorted atom order
__global__ void k_nl_cell_bounds(const int* __restrict__ sorted_cell, int n_atoms, int* __restrict__ cell_start,
                                 int* __restrict__ cell_end, const int* __restrict__ gate) {
    SPK_PDL_ENTER();
    if (grid_gated_off(gate)) return;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_atoms) return;
    const int c = sorted_cell[p];
    if (p == 0 || sorted_cell[p - 1] != c) cell_start[c] = p;
    if (p == n_atoms - 1 || sorted_cell[p + 1] != c) cell_end[c] = p + 1;
}

}  // namespace

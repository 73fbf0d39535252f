/*
 * spk_b200.h -- C ABI of the H100-native (sm_90a) message-passing hot path for SchNetPack models.
 *
 * The reference (atomistic-machine-learning/schnetpack @ 4c967da) has NO native interface for this path: every op is
 * an ATen kernel dispatched from Python (SURVEY.md section 2, "CUDA kernel inventory: empty").  The entry points below
 * are therefore what a ctypes binding inside the reference's own nn.Modules would bind (INTEGRATION.md shows the stub);
 * each one cites the reference Python it replaces (paths relative to /root/reference/src/schnetpack).
 *
 * Conventions (SURVEY.md section 8b):
 *   - every pointer is a DEVICE pointer to contiguous row-major data; floats are fp32, graph indices int32,
 *     user-facing neighbour indices (idx_i/idx_j/idx_m/Z) int64 exactly as the reference's tensors;
 *   - the caller owns every buffer (outputs and workspaces included); the library never allocates, never
 *     synchronises, keeps no global mutable state (it reads no environment
 *     variables; per-device launch attributes are cached) and only enqueues work on the given stream (graph-capturable);
 *   - return value: 0 = ok, SPK_ERR_ARG (-1) bad argument, SPK_ERR_UNSUPPORTED (-2) shape outside the compiled
 *     templates, -(1000 + cudaError_t) if a launch failed.  Nothing throws.
 *   - F = n_atom_basis (multiple of 32, <= 256), n_rbf <= 32, KP = SPK_KP(n_rbf) = n_rbf rounded up to 4.
 */
#ifndef SPK_B200_H
#define SPK_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* spk_stream_t; /* cudaStream_t */

#define SPK_OK 0
#define SPK_ERR_ARG (-1)
#define SPK_ERR_UNSUPPORTED (-2)

#define SPK_ACT_NONE 0
#define SPK_ACT_SILU 1 /* torch.nn.functional.silu            (PaiNN, Atomwise)  */
#define SPK_ACT_SSP 2  /* nn/activations.py:9-22 shifted_softplus (SchNet)        */
#define SPK_ACT_GIVEN 3      /* a_act only: a_pre already holds act'(pre) (saved by the forward layer, see below)  */
#define SPK_SAVE_DERIV 0x10  /* OR-ed into `act`: y_pre receives act'(pre) instead of the pre-activation, so the input-
                              * gradient layer multiplies by it without re-evaluating exp() (a_act = SPK_ACT_GIVEN)  */

#define SPK_RBF_GAUSSIAN 0 /* nn/radial.py:11-48  */
#define SPK_RBF_BESSEL 1   /* nn/radial.py:82-110 */

#define SPK_GEO_STRIDE 8 /* floats per edge in the geometry record: ux uy uz d fc dfc/dd 1/d 0 */
#define SPK_NRB(n_rbf) ((n_rbf) <= 20 ? 20 : 32)          /* radial-basis capacity of the compiled edge kernels */

int spk_version(void);

/* ---------------------------------------------------------------------------------------------------------------
 * Graph structure.  Replaces the implicit ordering assumptions of index_select / index_add_ in
 * nn/scatter.py:26-34, representation/painn.py:55-62, representation/schnet.py:65-67.
 *   rowptr[N+1], slot_j[E], slot_eid[E] : edges grouped by receiver idx_i (CSR).  Slot s of row i holds the sender
 *       slot_j[s] and the position slot_eid[s] of that edge in the caller's idx_i/idx_j arrays.  If idx_i is already
 *       sorted (reference collate order) slots are the identity permutation; otherwise a stable grouping is built.
 *   sptr[N+1], pos_slot[E], pos_i[E]    : the same edges grouped by sender idx_j (ascending slot inside a group).
 *   status[4] (device int32): [0]=1 if idx_i was sorted, [1]=number of out-of-range indices (must be 0; otherwise
 *       rowptr and sptr are zeroed = an empty graph, so no consumer gathers through unwritten slots),
 *       [2]=max receiver degree, [3]=max sender degree.
 *   workspace: spk_graph_workspace_bytes(N, E) bytes.
 * ------------------------------------------------------------------------------------------------------------- */
size_t spk_graph_workspace_bytes(int64_t n_atoms, int64_t n_edges);
int spk_graph_build(const int64_t* idx_i, const int64_t* idx_j, int64_t n_atoms, int64_t n_edges, int32_t* rowptr,
                    int32_t* slot_j, int32_t* slot_eid, int32_t* sptr, int32_t* pos_slot, int32_t* pos_i,
                    int32_t* status, void* workspace, size_t workspace_bytes, spk_stream_t stream);

/* The same views over the ACTIVE edges only: an edge is kept iff |r_ij[e]| < cutoff, i.e. iff the cosine cutoff does not
 * zero its message (nn/cutoff.py:30-32) -- padded neighbour lists (slots at distance >= cutoff) then cost nothing in the
 * edge kernels.  rowptr[n_atoms] (device) is the number of kept edges; slot arrays are filled for [0, rowptr[n_atoms]) and
 * slot_eid still points into the caller's full edge arrays.  r_ij [E,3] fp32. */
int spk_graph_build_active(const int64_t* idx_i, const int64_t* idx_j, const float* r_ij, float cutoff, int64_t n_atoms,
                           int64_t n_edges, int32_t* rowptr, int32_t* slot_j, int32_t* slot_eid, int32_t* sptr,
                           int32_t* pos_slot, int32_t* pos_i, int32_t* status, void* workspace, size_t workspace_bytes,
                           spk_stream_t stream);

/* mol_ptr[B+1] from the sorted system index idx_m (atomistic/atomwise.py:79-81 uses idx_m with index_add). */
int spk_segment_ptr(const int64_t* idx_m, int64_t n_atoms, int64_t n_mol, int32_t* mol_ptr, spk_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Geometry.  atomistic/distances.py:14-26 (PairwiseDistances), representation/painn.py:227-230,
 * representation/schnet.py:156-158, nn/radial.py, nn/cutoff.py:14-33.
 * ------------------------------------------------------------------------------------------------------------- */
/* Rij[e] = R[idx_j[e]] - R[idx_i[e]] + offsets[e]; an edge with an index outside [0, n_atoms) yields NaN (no OOB read) */
int spk_pairwise_fwd(const float* R, const int64_t* idx_i, const int64_t* idx_j, const float* offsets, int64_t n_atoms,
                     int64_t n_edges, float* r_ij, spk_stream_t stream);
/* dE/dR[a] = sum_{e: j(e)=a} g[e] - sum_{e: i(e)=a} g[e]   (deterministic, no atomics); out = sign * that */
int spk_pairwise_bwd(const float* g_rij, const int32_t* rowptr, const int32_t* slot_eid, const int32_t* sptr,
                     const int32_t* pos_slot, int64_t n_atoms, float sign, float* g_R, spk_stream_t stream);
/* per CSR slot s (edge slot_eid[s]): phi[s,0:n_rbf] radial basis (zero padded to KP), dphi = d phi/dd,
 * geo[s] = (ux, uy, uz, d, fc, dfc/dd, 1/d, 0).  rbf_p0/p1 = offsets/widths (gaussian) or freqs/NULL (bessel).
 * n_active (nullable, device): number of slots that exist (rowptr[n_atoms] of spk_graph_build_active); slots past it are
 * left untouched. */
int spk_edge_geometry(const float* r_ij, const int32_t* slot_eid, int64_t n_edges, int rbf_kind, int n_rbf,
                      const float* rbf_p0, const float* rbf_p1, float cutoff, const int32_t* n_active, float* phi,
                      float* dphi, float* geo, spk_stream_t stream);
/* standalone radial basis / cutoff / activation (nn.GaussianRBF, nn.BesselRBF, nn.CosineCutoff, shifted_softplus
 * forward + derivative, used by the nn.* module mirrors).  d: [n]; out: [n, n_rbf]; dout nullable */
int spk_rbf_fwd(const float* d, int64_t n, int rbf_kind, int n_rbf, const float* rbf_p0, const float* rbf_p1,
                float* out, float* dout, spk_stream_t stream);
int spk_cosine_cutoff_fwd(const float* d, int64_t n, float cutoff, float* out, float* dout, spk_stream_t stream);
int spk_act_fwd(const float* x, int64_t n, int act, float* y, float* dy, spk_stream_t stream);
/* out[a, :] = table[Z[a], :]   (nn.Embedding in representation/painn.py:239, schnet.py:161); Z outside [0, n_rows)
 * (nn.Embedding raises) gives a NaN row */
int spk_embedding(const float* table, const int64_t* Z, int64_t n_atoms, int F, int n_rows, float* out,
                  spk_stream_t stream);
/* out[idx[r], :] += x[r, :] for sorted-or-not idx via a row-pointer (deterministic): generic nn/scatter.py:7-34.
 * rowptr/slot_eid from spk_graph_build-style grouping of idx.  out[n_out, C] is fully overwritten. */
int spk_segment_sum(const float* x, const int32_t* rowptr, const int32_t* slot_eid, int64_t n_out, int C, float* out,
                    spk_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Dense layers.  nn/base.py:52-55 (Dense.forward = activation(F.linear(x, W, b))).
 *   Y[M,N] = act( A[M,K] * B[K,N] + bias[N] ) + addend[M,N]
 * B is the TRANSPOSED torch weight (W^T, [in,out] row-major) for a forward layer, or the weight itself for the
 * input-gradient of a layer ( gX = (gY .* act'(pre)) W ).  If a_pre != NULL the A operand is multiplied on load by
 * act'(a_pre) with activation a_act (the backward prologue).  y_pre (nullable) receives the pre-activation.
 * ------------------------------------------------------------------------------------------------------------- */
int spk_dense(const float* A, int64_t M, int K, int64_t lda, const float* a_pre, int a_act, const float* B, int N,
              const float* bias, int act, const float* addend, int64_t ld_add, float* Y, int64_t ldy, float* y_pre,
              spk_stream_t stream);

/* Contract of every PACKED operand (spk_tc_pack_weight, spk_painn_pack_filter, spk_schnet_pack_filter): the packed buffer is
 * a static operand.  The tensor-core kernels fetch it by TMA BEFORE their programmatic-launch dependency wait, so it must be
 * written only by these pack entry points (whose kernels never release their dependents early) or be complete before the
 * preceding kernels of the stream were launched; do not overwrite it with other kernels while evaluations are in flight. */
/* Same layer on the Hopper tensor cores (wgmma) with 3xTF32 error compensation (fp32-grade results: split accumulators, K-tile
 * draining; see csrc/gemm_tc.cu).  The weight the A rows are contracted with -- the torch weight [N,K] itself for a
 * forward layer, its transpose for the input-gradient -- is packed once by spk_tc_pack_weight into per-(64-row, 16-column)
 * operand tiles [tf32_round(W) | W - tf32_round(W)] laid out exactly as the kernel's shared-memory wgmma operand, so one TMA
 * bulk copy stages a tile.  Requirements: K, N, lda, ldy, ld_add multiples of 4, 16 B-aligned pointers, and at most one of
 * (a_act, act) active; otherwise SPK_ERR_UNSUPPORTED is returned and the caller uses spk_dense. */
size_t spk_tc_packed_floats(int N, int K);
int spk_tc_pack_weight(const float* W, int N, int K, float* packed, spk_stream_t stream);
int spk_dense_tc(const float* A, int64_t M, int K, int64_t lda, const float* a_pre, int a_act, const float* W_packed,
                 int N, const float* bias, int act, const float* addend, int64_t ld_add, float* Y, int64_t ldy,
                 float* y_pre, spk_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * PaiNN.  representation/painn.py:31-67 (PaiNNInteraction.forward) and :92-117 (PaiNNMixing.forward).
 * ------------------------------------------------------------------------------------------------------------- */
/* Fused per-edge kernel of one interaction block (painn.py:55-65 + the filter of :232-236 recomputed on the fly):
 *   W_s   = fc_s * (bf + phi_s Wf^T)                       [3F]   (never materialised)
 *   q_out[i]  = q[i]  + sum_{s in row i} W_s[0:F]   * x[j_s, 0:F]
 *   mu_out[i] = mu[i] + sum_{s in row i} W_s[F:2F]  * x[j_s, F:2F] (x) u_s + W_s[2F:3F] * x[j_s, 2F:3F] * mu[j_s]
 * x = interatomic_context_net(q) [N,3F]; mu [N,3,F] may be NULL (== zeros, first block); wf [3F, n_rbf] and bf [3F]
 * are this block's rows of filter_net.{weight,bias}.  q_out may alias q; mu_out must not alias mu. */
int spk_painn_edge_fwd(const float* x, const float* mu, const float* q, const float* phi, const float* geo,
                       const int32_t* rowptr, const int32_t* slot_j, const float* wf, const float* bf, int64_t n_atoms,
                       int64_t n_edges, int F, int n_rbf, float* q_out, float* mu_out, spk_stream_t stream);
/* Reverse of the above grouped by SENDER (no atomics): given g_q = dE/dq_out [N,F], g_mu = dE/dmu_out [N,3,F]:
 *   g_x[j]     = sum_{edges with sender j} ...                                   [N,3F]  (overwritten)
 *   g_mu_in[j] = g_mu[j] + sum ...                                               [N,3,F] (nullable when mu == NULL)
 *   g_rij[eid] (+)= dE/dr_ij through d (phi, fc) and u                           [E,3]   (accumulate != 0 -> +=)
 * The residual dE/dq_in = g_q is the caller's (identity).  */
int spk_painn_edge_bwd(const float* x, const float* mu, const float* g_q, const float* g_mu, const float* phi,
                       const float* dphi, const float* geo, const int32_t* sptr, const int32_t* pos_slot,
                       const int32_t* pos_i, const int32_t* slot_eid, const float* wf, const float* bf,
                       int64_t n_atoms, int64_t n_edges, int F, int n_rbf, float* g_x, float* g_mu_in, float* g_rij,
                       int accumulate, spk_stream_t stream);
/* Tensor-core variant of spk_painn_edge_fwd (csrc/painn_tc.cu): the filter W = fc * (phi . w^T + b) of a chunk of edges is
 * computed by a producer warpgroup with 3xTF32 wgmma (channels on the M side) and handed to the gather/accumulate warps as
 * a filter tile in shared memory, so they read their channel's filter values instead of recomputing them from
 * warp-broadcast shared-memory loads (the streaming kernel is bound by the load/store unit).
 * wf_packed = spk_painn_pack_filter(wf, bf) (hi/lo operand tiles, spk_painn_filter_packed_floats() floats).  Same results
 * as spk_painn_edge_fwd to fp32 rounding.  Returns SPK_ERR_UNSUPPORTED unless F == 128, n_rbf <= 31 and n_edges > 0
 * (the caller then uses spk_painn_edge_fwd). */
size_t spk_painn_filter_packed_floats(void);
int spk_painn_pack_filter(const float* wf, const float* bf, int F, int n_rbf, float* packed, spk_stream_t stream);
int spk_painn_edge_fwd_tc(const float* x, const float* mu, const float* q, const float* phi, const float* geo,
                          const int32_t* rowptr, const int32_t* slot_j, const float* wf_packed, int64_t n_atoms,
                          int64_t n_edges, int F, int n_rbf, float* q_out, float* mu_out, spk_stream_t stream);
/* Tensor-core variant of spk_painn_edge_bwd: one operand of 64 rows per chunk of 32 edges, rows 0..31 = fc [phi | 1],
 * rows 32..63 = dfc [phi | 1] + fc [dphi | 0], so the same 27 MMAs produce W and dW/dd for the 8 edges of each of the 4
 * sender groups.  Same outputs as spk_painn_edge_bwd to fp32 rounding; SPK_ERR_UNSUPPORTED under the conditions of
 * spk_painn_edge_fwd_tc. */
int spk_painn_edge_bwd_tc(const float* x, const float* mu, const float* g_q, const float* g_mu, const float* phi,
                          const float* dphi, const float* geo, const int32_t* sptr, const int32_t* pos_slot,
                          const int32_t* pos_i, const int32_t* slot_eid, const float* wf_packed, int64_t n_atoms,
                          int64_t n_edges, int F, int n_rbf, float* g_x, float* g_mu_in, float* g_rij, int accumulate,
                          spk_stream_t stream);
/* Block-level interaction with a caller-supplied, materialised filter -- PaiNNInteraction.forward(q, mu, Wij, dir_ij, idx_i,
 * idx_j, n_atoms), painn.py:31-67 (csrc/painn_block.cu).  Wij [E,3F] and dir [E,3] are in the CALLER's edge order (looked
 * up through slot_eid); x = interatomic_context_net(q) [N,3F]; mu [N,3,F] required.  Reverse: g_x [N,3F], g_mu_in [N,3,F]
 * (= g_mu + ...), g_W [E,3F], g_dir [E,3] in the caller's edge order, all overwritten. */
int spk_painn_edge_wij_fwd(const float* x, const float* mu, const float* q, const float* Wij, const float* dir,
                           const int32_t* rowptr, const int32_t* slot_j, const int32_t* slot_eid, int64_t n_atoms,
                           int64_t n_edges, int F, float* q_out, float* mu_out, spk_stream_t stream);
int spk_painn_edge_wij_bwd(const float* x, const float* mu, const float* g_q, const float* g_mu, const float* Wij,
                           const float* dir, const int32_t* sptr, const int32_t* pos_slot, const int32_t* pos_i,
                           const int32_t* slot_eid, int64_t n_atoms, int64_t n_edges, int F, float* g_x, float* g_mu_in,
                           float* g_W, float* g_dir, spk_stream_t stream);
/* painn.py:104-107: ctx[a] = [ q[a] | sqrt(sum_d V[a,d]^2 + eps) ], VW = mu_channel_mix(mu) [N,3,2F] */
int spk_painn_mix_ctx(const float* q, const float* VW, int64_t n_atoms, int F, float eps, float* ctx,
                      spk_stream_t stream);
/* painn.py:110-116: q_out = q + s1 + s3 * sum_d V_d W_d ; mu_out[d] = mu[d] + s2 * W_d ; s [N,3F] */
int spk_painn_mix_update(const float* q, const float* mu, const float* s, const float* VW, int64_t n_atoms, int F,
                         float* q_out, float* mu_out, spk_stream_t stream);
/* reverse of mix_update: g_s [N,3F]; g_VW [N,3,2F] (without the norm path) */
int spk_painn_mix_update_bwd(const float* g_q, const float* g_mu, const float* s, const float* VW, int64_t n_atoms,
                             int F, float* g_s, float* g_VW, spk_stream_t stream);
/* reverse of mix_ctx: g_q_out = g_q + g_ctx[:, :F]; g_VW[:, d, :F] += g_ctx[:, F:] * V_d / n */
int spk_painn_mix_ctx_bwd(const float* g_ctx, const float* g_q, const float* VW, int64_t n_atoms, int F, float eps,
                          float* g_q_out, float* g_VW, spk_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * SchNet.  representation/schnet.py:41-70 (SchNetInteraction.forward).
 * ------------------------------------------------------------------------------------------------------------- */
/* continuous-filter convolution (schnet.py:62-67): m[i] = sum_{s in row i} h[j_s] * Wraw[s] * fc_s ; Wraw [E,F] is
 * the filter-network output per CSR slot. */
int spk_cfconv_fwd(const float* h, const float* w_raw, const float* geo, const int32_t* rowptr, const int32_t* slot_j,
                   int64_t n_atoms, int64_t n_edges, int F, float* m, spk_stream_t stream);
/* The whole interaction-block forward edge pipeline fused, filter network on wgmma (csrc/schnet_tc.cu):
 *   m[i] = sum_{s in row i} h[j_s] * ( W1 act(W0 phi_s + b0) + b1 ) * fc_s          schnet.py:61-67
 * filter_packed = spk_schnet_pack_filter(filter_network.0.{weight,bias}, filter_network.1.weight) (hi|lo operand tiles,
 * spk_schnet_filter_packed_floats() floats); b1 = filter_network.1.bias; act = SPK_ACT_SSP | SPK_ACT_SILU | SPK_ACT_NONE.
 * rowptr may come from spk_graph_build_active (rowptr[n_atoms] slots exist; n_edges is only the capacity of the arrays).
 * F == n_filters == 128 and n_rbf <= 31, otherwise SPK_ERR_UNSUPPORTED (the caller runs the materialised pipeline). */
size_t spk_schnet_filter_packed_floats(void);
int spk_schnet_pack_filter(const float* w0, const float* b0, const float* w1, int F, int n_rbf, float* packed,
                           spk_stream_t stream);
int spk_schnet_cfconv_fwd_tc(const float* h, const float* phi, const float* geo, const int32_t* rowptr,
                             const int32_t* slot_j, const float* filter_packed, const float* b1, int act, int64_t n_atoms,
                             int64_t n_edges, int F, int n_rbf, float* m, spk_stream_t stream);
/* reverse grouped by sender: g_h[j] = sum W fc g_m[i];  g_wraw[s] = h[j] g_m[i] fc_s;
 * g_fc[s] = sum_c h[j,c] g_m[i,c] Wraw[s,c] */
int spk_cfconv_bwd(const float* h, const float* w_raw, const float* geo, const float* g_m, const int32_t* sptr,
                   const int32_t* pos_slot, const int32_t* pos_i, int64_t n_atoms, int64_t n_edges, int F, float* g_h,
                   float* g_wraw, float* g_fc, spk_stream_t stream);
/* g_rij[eid] (+)= ( sum_k g_phi[s,k] dphi[s,k] + g_fc[s] dfc_s ) * u_s      (d-only dependence of SchNet) */
int spk_radial_bwd(const float* g_phi, const float* g_fc, const float* dphi, const float* geo, const int32_t* slot_eid,
                   int64_t n_edges, int n_rbf, float* g_rij, int accumulate, spk_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Atomwise head.  atomistic/atomwise.py:69-88: y = outnet(q); E[m] = sum_{a in m} y[a].
 * ------------------------------------------------------------------------------------------------------------- */
/* y[a] = hid[a,:] . w1 + b1 ; energy[m] = sum_{a in mol m} y[a]   (hid = silu(Dense_0(q)) [N,H]); y nullable */
int spk_atomwise_out(const float* hid, const float* w1, const float* b1, const int32_t* mol_ptr, int64_t n_atoms,
                     int64_t n_mol, int H, float* y, float* energy, spk_stream_t stream);
/* g_hid[a,:] = g_energy[mol(a)] * w1   (g_energy nullable == ones) */
int spk_atomwise_out_bwd(const float* g_energy, const int64_t* idx_m, const float* w1, int64_t n_atoms, int H,
                         float* g_hid, spk_stream_t stream);

/* elementwise helpers for residual streams: out = a + b (b nullable -> copy), may alias */
int spk_add(const float* a, const float* b, int64_t n, float* out, spk_stream_t stream);

/* ---- "next" row f1: device-resident neighbour list (replaces the host round trip of md/neighborlist_md.py:129,213-232 and
 * the ASE / matscipy / vesin / torch builders of transform/neighborlist.py:213-286,428-553) ---------------------------------
 * Linked-cell search per system of a collated batch.  Listed: every (i, j, S) with |R[j] - R[i] + S @ cell| < cutoff, S
 * integer with S_a = 0 on non-periodic axes, except (i == j, S == 0); offsets = S @ cell (fp32); rows sorted by idx_i, a row
 * in traversal order (deterministic; compare after the canonical (i, j, S) sort as the reference's tests do).
 *   R [n_atoms,3] fp32, cell [n_sys,3,3] fp32 (rows = lattice vectors; ignored where pbc is all zero), pbc [n_sys,3] uint8,
 *   sys_ptr [n_sys+1] int32 = first atom of every system (spk_segment_ptr).
 *   idx_i, idx_j [capacity] int64, offsets [capacity,3] fp32, shifts [capacity,3] int32 (nullable).
 *   n_pairs [2] int64 on the DEVICE: [0] = pairs found, [1] = 1 if they exceeded `capacity` (then only the first
 *   `capacity` were written).  pad != 0 spreads the unused capacity over the rows as self pairs (i, i) at distance
 *   2 * cutoff appended to each row -- outside the cutoff, so they contribute nothing to energies or forces, idx_i stays
 *   sorted and no row grows long -- which lets a caller run a fixed-size edge list without ever reading n_pairs on the host
 *   (CUDA-graph capturable MD step).  Without pad the pairs are contiguous in [0, n_pairs).  capacity == 0 only counts.
 * Enqueue-only on `stream`; workspace of spk_neighbor_list_workspace_bytes(n_atoms, n_sys) bytes. */
size_t spk_neighbor_list_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_neighbor_list(const float* R, const float* cell, const uint8_t* pbc, const int32_t* sys_ptr, int64_t n_atoms,
                      int64_t n_sys, float cutoff, int64_t capacity, int pad, int64_t* idx_i, int64_t* idx_j,
                      float* offsets, int32_t* shifts, int64_t* n_pairs, void* workspace, size_t workspace_bytes,
                      spk_stream_t stream);

/* ---- row e: halo exchange of ghost-atom rows over NVLink peer memory (csrc/halo.cu).  peer_base[world] (device array) holds
 * every rank's symmetric buffer address as mapped into THIS process (CUDA IPC / torch symmetric memory); the caller has
 * enqueued a cross-rank barrier after the owners wrote their rows.
 *   spk_halo_pull      ghost[k, :] = peer[ghost_rank[k]][ghost_row[k], :]          rows of row_floats floats
 *   spk_halo_pull_add  g_rows[rows[k], :] += sum_{e in [entry_ptr[k], entry_ptr[k+1])} peer[entry_rank[e]][entry_pos[e], :]
 *                      (entries of a row in ascending peer order: deterministic reverse halo, no atomics) */
int spk_halo_pull(float* ghost, const uint64_t* peer_base, const int32_t* ghost_rank, const int32_t* ghost_row,
                  int64_t n_ghost, int row_floats, spk_stream_t stream);
int spk_halo_pull_add(float* g_rows, const uint64_t* peer_base, const int32_t* rows, const int32_t* entry_ptr,
                      const int32_t* entry_rank, const int32_t* entry_pos, int64_t n_listed, int row_floats,
                      spk_stream_t stream);

/* ---- "next" row f2: velocity-Verlet update of the device-resident MD state (md/integrators.py:59-70,97-110;
 * unit handling of md/calculators/base_calculator.py:96,120-152).  momenta [N,3] += 1/2 dt * forces * force_conversion; with
 * drift != 0 also positions [N,3] += dt * momenta / masses [N] and, if given, model_positions = positions *
 * position_conversion (the array the next force evaluation reads).  All in place, enqueue-only. */
int spk_md_velocity_verlet(float* momenta, float* positions, float* model_positions, const float* forces,
                           const float* masses, int64_t n_atoms, float dt, float force_conversion,
                           float position_conversion, int drift, spk_stream_t stream);

/* ---- thermostats of the device MD step (md/simulation_hooks/thermostats.py:149-513, md/system.py:374-421).  Applied to the
 * momenta before the first and after the second half kick (md/simulator.py:127-150).  Systems are those of a collated batch:
 * idx_m [n_atoms] int64 sorted, sys_ptr [n_sys+1] int32 (spk_segment_ptr); masses [n_atoms] fp32; momenta [n_atoms,3] fp32
 * in place.  Every per-system sum is accumulated in fp64 in a fixed order (no atomics): bitwise reproducible.
 * workspace: spk_md_thermostat_workspace_bytes(n_atoms, n_sys) bytes, 8-byte aligned, no initialisation needed.
 *   spk_md_kinetic_energy  ke[s] = 1/2 sum_{a in s} |p_a|^2 / m_a, temperature[s] = 2 ke[s] / (3 n_s kB)  (fp64, nullable)
 *   spk_md_berendsen       p *= sqrt(1 + dt_over_tau (temperature_bath / T_s - 1)) per system (unchanged where T_s = 0)
 *   spk_md_nhc             Nose-Hoover chains (:398-468) propagated with params, p *= the chain's scaling.  Chain state
 *                          chain_v, chain_f, chain_m [n_chain, chain_length] fp64, n_chain = n_sys, or 3 n_atoms when
 *                          massive (one chain per degree of freedom, row 3a+d; idx_m / sys_ptr / workspace unused then).
 *                          chain_m holds the thermostat masses (:375-396); velocities and forces start at zero and are
 *                          advanced in place.
 *   spk_md_langevin        p = c1 p + c2 sqrt(m kb_temperature) xi, xi ~ N(0,1) from Philox4x32-10 with key = seed and
 *                          counter = (atom index, counter[0]) through Box-Muller (normals 0..2 of the draw for x, y, z).
 *                          counter [2] uint64 on the DEVICE: [0] = application index, advanced by one in stream order by
 *                          every call (so a replayed graph draws fresh noise each time), [1] = 0 (internal ticket).
 *   spk_philox4x32_10      out[4 i + k] = word k of the Philox4x32-10 draw for element i, application counter[0], key
 *                          seed (counter not advanced): the raw bits behind spk_md_langevin.
 * Per-system bath temperatures (DESIGN.md section 25): kb_temperature_sys [n_sys] fp64 on the device holds kB T_s of every
 * system.  spk_md_langevin_per_system is spk_md_langevin with kB T_s of the atom's system idx_m[a]; spk_md_nhc_per_system
 * is spk_md_nhc with every chain forced at kB T_s of its system (of its atom's system when massive; idx_m is read then),
 * params->kb_temperature unused.  The chain masses chain_m must be built from the same kB T_s.  With every kB T_s equal to
 * kb_temperature they give bitwise the results of the scalar entry points. */
typedef struct {
    int32_t chain_length;  /* >= 1 */
    int32_t multi_step;    /* >= 1 */
    int32_t order;         /* Yoshida-Suzuki order 3, 5 or 7 = entries of time_step used */
    int32_t massive;       /* 0: one chain per system, 1: one chain per degree of freedom */
    double kb_temperature; /* kB * T_bath in MD energy units */
    double time_step[7];   /* dt * w_k / multi_step, w = Yoshida-Suzuki weights (md/utils/thermostat_utils.py:18-44) */
} spk_nhc_params_t;

size_t spk_md_thermostat_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_md_kinetic_energy(const float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                          int64_t n_atoms, int64_t n_sys, double kB, double* ke, double* temperature, void* workspace,
                          size_t workspace_bytes, spk_stream_t stream);
int spk_md_berendsen(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                     int64_t n_sys, double kB, double dt_over_tau, double temperature_bath, void* workspace,
                     size_t workspace_bytes, spk_stream_t stream);
int spk_md_nhc(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
               int64_t n_sys, const spk_nhc_params_t* params, double* chain_v, double* chain_f, const double* chain_m,
               void* workspace, size_t workspace_bytes, spk_stream_t stream);
int spk_md_langevin(float* momenta, const float* masses, int64_t n_atoms, double c1, double c2, double kb_temperature,
                    uint64_t seed, uint64_t* counter, spk_stream_t stream);
int spk_philox4x32_10(uint64_t seed, const uint64_t* counter, int64_t n, uint32_t* out, spk_stream_t stream);
int spk_md_langevin_per_system(float* momenta, const float* masses, const int64_t* idx_m, int64_t n_atoms, double c1,
                               double c2, const double* kb_temperature_sys, uint64_t seed, uint64_t* counter,
                               spk_stream_t stream);
int spk_md_nhc_per_system(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                          int64_t n_atoms, int64_t n_sys, const spk_nhc_params_t* params,
                          const double* kb_temperature_sys, double* chain_v, double* chain_f, const double* chain_m,
                          void* workspace, size_t workspace_bytes, spk_stream_t stream);

/* ---- per-system virial (csrc/geometry.cu): W[m][b][a] = sum_{e in m} g_rij[e][b] * r_ij[e][a] in fp64, the strain
 * derivative dE/d(strain) of atomistic/response.py:78-90 (Strain maps r_e -> r_e (1 + strain^T)); the stress is W / V.
 * The edges of system m are the receiver slots [rowptr[sys_ptr[m]], rowptr[sys_ptr[m+1]]) of the graph view of
 * spk_graph_build, mapped to edge ids by slot_eid; sys_ptr [n_sys+1] int32 = first atom of every system
 * (spk_segment_ptr).  g_rij, r_ij [n_edges,3] fp32 in edge order; virial [n_sys,3,3] fp64, overwritten.  Reduced with
 * fixed-shape CTA partials and an ordered per-system pass (no atomics): bitwise reproducible for any mix of system sizes.
 * workspace: spk_pairwise_virial_workspace_bytes(n_edges, n_sys) bytes, 8-byte aligned, no initialisation needed. */
size_t spk_pairwise_virial_workspace_bytes(int64_t n_edges, int64_t n_sys);
int spk_pairwise_virial(const float* g_rij, const float* r_ij, const int32_t* rowptr, const int32_t* slot_eid,
                        const int32_t* sys_ptr, int64_t n_edges, int64_t n_sys, double* virial, void* workspace,
                        size_t workspace_bytes, spk_stream_t stream);

/* ---- Nose-Hoover-chain barostats of the device MD step (csrc/barostat.cu; md/simulation_hooks/barostats.py:162-927 with
 * md/integrators.py:232-263 NPTVelocityVerlet).  Systems, masses and momenta as for the thermostats above; positions
 * [n_atoms,3] fp32 in MD units; cell [n_sys,3,3] fp64 in MD units (rows = lattice vectors).  One step (simulator.py:124-150):
 * thermostat, kick, half_step, main_step, forces + virial, half_step, kick, thermostat.
 * workspace: spk_md_barostat_workspace_bytes(n_atoms, n_sys) bytes, 8-byte aligned, no initialisation needed; the operators
 * of half_step / main_step live there between their two launches only.
 *   spk_md_kinetic_energy_tensor  ke_tensor[s] = 1/2 sum_{a in s} p_a p_a^T / m_a  [n_sys,3,3] fp64 (system.py:389-404)
 *   spk_md_barostat_thermostat    _update_thermostat (:408-481): the particle chains (per system, or per degree of freedom
 *                                 when massive) scale the momenta, the cell chain (per system) scales b_v
 *   spk_md_barostat_kick          _update_barostat (:604-631 isotropic, :822-842 anisotropic): b_f from the pressure with
 *                                 stress = virial_scale * virial / V (virial [n_sys,3,3] fp64, V = det(cell)), then
 *                                 b_v += 1/2 dt b_f
 *   spk_md_barostat_half_step     propagate_half_step (:661-686, :885-926): p = p A + 1/2 dt (forces * force_conversion) B
 *   spk_md_barostat_main_step     propagate_main_step (:633-659, :844-883): x = x A + dt (p / m) B, cell scaled (isotropic:
 *                                 cell * exp(dt b_v); anisotropic: cell @ A), model_cell [n_sys,3,3] fp32 = cell *
 *                                 position_conversion and model_positions = x * position_conversion (both nullable).
 * The anisotropic operators come from a per-system fp64 Jacobi eigendecomposition of b_v that reads its upper triangle (as
 * torch.symeig(upper=True) did).  sinh(x)/x is md/utils/thermostat_utils.py:181-201 StableSinhDiv exactly as written. */
typedef struct {
    int32_t anisotropic;     /* 0: one cell velocity per system (b_v, b_f [n_sys]); 1: 3x3 (b_v, b_f [n_sys,3,3]) */
    int32_t massive;         /* 0: one particle chain per system; 1: one per degree of freedom (row 3a+d) */
    int32_t chain_length;    /* >= 1, both chains */
    int32_t multi_step;      /* >= 1 */
    int32_t order;           /* Yoshida-Suzuki order 3, 5 or 7 = entries of ys_time_step used */
    int32_t reserved;
    double kb_temperature;   /* kB * T_bath in MD energy units */
    double time_step;        /* dt in MD time units */
    double target_pressure;  /* P0 in MD pressure units (energy / length^3) */
    double ys_time_step[7];  /* dt * w_k / multi_step */
    double* t_v;             /* particle chains [n_chain, chain_length] fp64: velocities, forces, masses */
    double* t_f;
    const double* t_m;
    double* c_v;             /* cell chain [n_sys, chain_length] fp64 */
    double* c_f;
    const double* c_m;
    double* b_v;             /* cell velocities, forces [n_sys] or [n_sys,3,3], masses [n_sys] fp64 */
    double* b_f;
    const double* b_m;
} spk_nhc_barostat_t;

size_t spk_md_barostat_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_md_kinetic_energy_tensor(const float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                                 int64_t n_atoms, int64_t n_sys, double* ke_tensor, void* workspace,
                                 size_t workspace_bytes, spk_stream_t stream);
int spk_md_barostat_thermostat(const spk_nhc_barostat_t* barostat, float* momenta, const float* masses,
                               const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys,
                               void* workspace, size_t workspace_bytes, spk_stream_t stream);
int spk_md_barostat_kick(const spk_nhc_barostat_t* barostat, const float* momenta, const float* masses,
                         const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, const double* cell,
                         const double* virial, double virial_scale, void* workspace, size_t workspace_bytes,
                         spk_stream_t stream);
int spk_md_barostat_half_step(const spk_nhc_barostat_t* barostat, float* momenta, const float* forces,
                              double force_conversion, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                              int64_t n_sys, void* workspace, size_t workspace_bytes, spk_stream_t stream);
int spk_md_barostat_main_step(const spk_nhc_barostat_t* barostat, float* positions, float* model_positions,
                              const float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                              int64_t n_atoms, int64_t n_sys, double* cell, float* model_cell, double position_conversion,
                              void* workspace, size_t workspace_bytes, spk_stream_t stream);

/* ---- ring-polymer MD of the device MD step (csrc/rpmd.cu; md/integrators.py:113-229 RingPolymer,
 * md/utils/normal_model_transformation.py, md/simulation_hooks/thermostats_rpmd.py:33-234,373-501).  Bead arrays
 * [n_beads, n_atoms, 3] fp32 in MD units, replica-major (bead r of atom a at row r n_atoms + a); masses [n_atoms] fp32 of
 * the base batch (one copy of every atom); 1 <= n_beads <= 64.  c_transform [n_beads, n_beads] fp64 on the device is the
 * normal-mode matrix C (modes = C beads, beads = C^T modes).  Arithmetic is fp64 with fp32 loads and stores.  Systems
 * (idx_m, sys_ptr, n_sys) are those of the base batch, as for the thermostats above; they are read by the global variants
 * only.  workspace: spk_rpmd_workspace_bytes(n_atoms, n_sys) bytes, 8-byte aligned, no initialisation needed.  One step
 * (md/simulator.py:124-150): thermostat, half kick on every bead (spk_md_velocity_verlet, drift = 0), main step, forces on
 * all beads, half kick, thermostat.
 *   spk_rpmd_normal_modes  out = C in (inverse = 0) or C^T in (inverse = 1) over the bead axis; may run in place
 *   spk_rpmd_main_step     integrators.py:221-230 per degree of freedom: (p~, x~) of mode k -> propagator [n_beads,2,2]
 *                          fp64 (p~' = U00 p~ + U01 m x~, x~' = U10 p~ / m + U11 x~); positions and momenta in place,
 *                          model_positions = positions * position_conversion (nullable)
 *   spk_rpmd_pile          p~_k = c1[k] p~_k + c2[k] sqrt(m kb_temperature) xi (kb_temperature = n_beads kB T; c1, c2
 *                          [n_beads] fp64 on the device) with xi from Philox4x32-10, key = seed, counter = (k n_atoms + a,
 *                          counter[0]), normals 0..2 of the draw for x, y, z; counter as for spk_md_langevin.  global != 0:
 *                          mode 0 is instead rescaled per system by the stochastic velocity rescaling factor of
 *                          thermostats_rpmd.py:160-189 from K0 = sum |p~_0|^2 / m, S = sum |xi_0|^2 and R = the x-noise of
 *                          the system's first atom (a system with K0 = 0 is left as it is)
 *   spk_rpmd_nhc           one Nose-Hoover chain per (mode, degree of freedom) on p~ (params->massive is ignored):
 *                          kinetic energy p~^2 / m, chain state chain_v, chain_f, chain_m [n_beads 3 n_atoms, chain_length]
 *                          fp64, row k 3 n_atoms + 3 a + d.  global != 0: mode 0 sees its system's sum |p~_0|^2 / m with
 *                          3 n_s degrees of freedom. */
size_t spk_rpmd_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_rpmd_normal_modes(const float* in, float* out, int64_t n_atoms, int32_t n_beads, const double* c_transform,
                          int32_t inverse, spk_stream_t stream);
int spk_rpmd_main_step(float* positions, float* momenta, float* model_positions, const float* masses, int64_t n_atoms,
                       int32_t n_beads, const double* c_transform, const double* propagator, double position_conversion,
                       spk_stream_t stream);
int spk_rpmd_pile(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                  int64_t n_sys, int32_t n_beads, const double* c_transform, const double* c1, const double* c2,
                  double kb_temperature, int32_t global, uint64_t seed, uint64_t* counter, void* workspace,
                  size_t workspace_bytes, spk_stream_t stream);
int spk_rpmd_nhc(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                 int64_t n_sys, int32_t n_beads, const double* c_transform, const spk_nhc_params_t* params, int32_t global,
                 double* chain_v, double* chain_f, const double* chain_m, void* workspace, size_t workspace_bytes,
                 spk_stream_t stream);

/* ---- GLE thermostats (csrc/rpmd.cu; md/simulation_hooks/thermostats.py:527-730 GLEThermostat, thermostats_rpmd.py:
 * 237-370 RPMDGLEThermostat and PIGLETThermostat).  Bead arrays, masses and c_transform as for spk_rpmd_pile; the
 * classical GLE is n_beads = 1 with c_transform = [[1.0]], which is exact in fp64.  state [n_beads 3 n_atoms, gle_dim]
 * fp64 holds the extended momenta of every (normal mode k, degree of freedom i) at row k 3 n_atoms + i;
 * 1 <= gle_dim <= 16.  c1, c2 [gle_dim, gle_dim] fp64 row-major on the device, or [n_beads, gle_dim, gle_dim] with
 * per_mode != 0 (PIGLET: mode k uses block k).  Noise column j of row (k, 3 a + d) is normal d of the Philox4x32-10 draw
 * with key seed and counter ((j n_beads + k) n_atoms + a, counter[0]); counter [2] as for spk_rpmd_pile, advanced by
 * every call.
 *   initial != 0   the free-particle-limit start (thermostats.py:687-701): state row = xi^T c2_k, no mass factor;
 *                  momenta and masses are not read (may be null)
 *   initial == 0   s[0] = p~; s = c1_k s + sqrt(m_a) c2_k xi (column-vector form of Ceriotti et al. 2010, where the
 *                  reference propagates s^T c1 = (c1^T s)^T); p~ = s[0] */
int spk_rpmd_gle(float* momenta, const float* masses, int64_t n_atoms, int32_t n_beads, const double* c_transform,
                 const double* c1, const double* c2, int32_t gle_dim, int32_t per_mode, double* state, uint64_t seed,
                 uint64_t* counter, int32_t initial, spk_stream_t stream);

/* ---- PILE barostat of ring-polymer NPT (csrc/rpmd.cu; md/simulation_hooks/barostats_rpmd.py:21-208 PILEBarostat with
 * md/integrators.py:266-305 NPTRingPolymer).  One isotropic cell momentum p_c of mass W per system of the base batch
 * (cell_momenta, cell_mass [n_sys] fp64); bead arrays, masses, idx_m and sys_ptr as for spk_rpmd_pile; cells and virial
 * [n_beads n_sys, 3, 3] fp64 per bead system, replica-major (bead r of system s is r n_sys + s).  workspace:
 * spk_rpmd_barostat_workspace_bytes(n_atoms, n_sys) bytes, 8-byte aligned, shared by the half and main step, no
 * initialisation needed.  Every sum is fixed-order fp64 without atomics.  One NPT-RPMD step (md/simulator.py:124-150)
 * is: thermostat, barostat_thermostat, half_step + spk_md_velocity_verlet(drift = 0), main_step, forces + virial,
 * half_step + spk_md_velocity_verlet(drift = 0), barostat_thermostat, thermostat.
 *   spk_rpmd_barostat_thermostat  p_c = c1 p_c + c2[s] xi (barostats_rpmd.py:101-110): xi is normal 0 of the Philox4x32-10
 *                                 draw with key seed and counter (s, counter[0]); counter [2] as for spk_rpmd_pile
 *   spk_rpmd_barostat_half_step   p_c += h c1 + h^2 c2 + h^3 c3, h = time_step / 2 (barostats_rpmd.py:164-205), from the
 *                                 momenta before the particle kick: c1 = 3 P (V_bar (P_c - target_pressure) +
 *                                 kb_temperature) with V_bar the bead mean of det(cell), P_c = -tr(bead mean of the stress)
 *                                 / 3 + 2 K_c / (3 V_bar), stress = virial_scale virial / det(cell), K_c from the bead mean
 *                                 of the momenta; c2 = sum F~_0 . p~_0 / m, c3 = sum |F~_0|^2 / (3 m) over normal mode 0 of
 *                                 the momenta and of the forces * force_conversion.  2 launches.
 *   spk_rpmd_barostat_main_step   a = exp(-dt p_c / W), b = StableSinhDiv(dt p_c / W) per system; p~_0 *= a, then x~_0 =
 *                                 x~_0 / a + b dt p~_0 / m; modes k >= 1 by the propagator as spk_rpmd_main_step; every
 *                                 bead copy of the cell divided by a, model_cells (nullable) = cells * position_conversion
 *                                 in fp32 (barostats_rpmd.py:113-162).  2 launches. */
size_t spk_rpmd_barostat_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_rpmd_barostat_thermostat(double* cell_momenta, int64_t n_sys, double c1, const double* c2, uint64_t seed,
                                 uint64_t* counter, spk_stream_t stream);
int spk_rpmd_barostat_half_step(const float* momenta, const float* forces, double force_conversion, const float* masses,
                                const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys,
                                int32_t n_beads, const double* c_transform, const double* cells, const double* virial,
                                double virial_scale, double target_pressure, double kb_temperature, double time_step,
                                const double* cell_mass, double* cell_momenta, void* workspace, size_t workspace_bytes,
                                spk_stream_t stream);
int spk_rpmd_barostat_main_step(float* positions, float* momenta, float* model_positions, const float* masses,
                                const int64_t* idx_m, int64_t n_atoms, int64_t n_sys, int32_t n_beads,
                                const double* c_transform, const double* propagator, double time_step,
                                const double* cell_momenta, const double* cell_mass, double* cells, float* model_cells,
                                double position_conversion, void* workspace, size_t workspace_bytes, spk_stream_t stream);

/* ---- SO3net (representation/so3net.py, nn/so3.py) -------------------------------------------------------------------
 * Features are [N, S, F] with S = (lmax+1)^2 rows s = l^2 + l + m per atom.  lmax <= 3, F % 4 == 0, F <= 256, any n_rbf;
 * otherwise SPK_ERR_UNSUPPORTED.  Clebsch-Gordan table and harmonics: csrc/so3_tables.cuh.
 *
 * Convolution of one interaction block over the receiver CSR (rowptr, slot_j) and the spk_edge_geometry records:
 *   y[i, so, f] = sum_{e -> i} sum_nz C * W[l(s1), f] * Y[s1](u_e) * x[j_e, s2, f],
 *   W[l, f] = fc_e * (phi_e . wf[l*F + f, :] + bf[l*F + f])                        (filter never stored) */
int spk_so3_conv_fwd(const float* x, const float* phi, const float* geo, const int32_t* rowptr, const int32_t* slot_j,
                     const float* wf, const float* bf, int64_t n_atoms, int64_t n_edges, int lmax, int F, int n_rbf,
                     float* y, spk_stream_t stream);
/* Reverse, grouped by sender (sptr, pos_slot, pos_i): g_x[j] = g_res[j] + sum_{e: j_e = j} dy/dx[j]^T g_y[i_e]
 * (g_x may be NULL: only g_rij; g_res may be NULL: no residual), g_rij[eid] (+)= dE/dr_ij through d and u. */
int spk_so3_conv_bwd(const float* x, const float* g_y, const float* phi, const float* dphi, const float* geo,
                     const int32_t* sptr, const int32_t* pos_slot, const int32_t* pos_i, const int32_t* slot_eid,
                     const float* wf, const float* bf, int64_t n_atoms, int64_t n_edges, int lmax, int F, int n_rbf,
                     const float* g_res, float* g_x, float* g_rij, int accumulate, spk_stream_t stream);
/* out = dx + SO3TensorProduct(dx, ddx), and its reverse (g_dx includes the identity term) */
int spk_so3_tp_fwd(const float* dx, const float* ddx, int64_t n_atoms, int lmax, int F, float* out, spk_stream_t stream);
int spk_so3_tp_bwd(const float* g, const float* dx, const float* ddx, int64_t n_atoms, int lmax, int F, float* g_dx,
                   float* g_ddx, spk_stream_t stream);
/* gate y[n, s, f] = x[n, s, f] * sigmoid(h[n, l(s)*F + f]); reverse: g_x for rows s >= 1, g_x0 [N,F] for row 0 (the
 * caller adds the gate layer's input gradient), g_h [N, (lmax+1) F] */
int spk_so3_gate_fwd(const float* x, const float* h, int64_t n_atoms, int lmax, int F, float* y, spk_stream_t stream);
int spk_so3_gate_bwd(const float* g_y, const float* x, const float* h, int64_t n_atoms, int lmax, int F, float* g_x,
                     float* g_x0, float* g_h, spk_stream_t stream);
/* out[n, s, f] = (src ? src[n, s, f] : 0) + (s == 0 ? v[n, f] : 0);  q[n, f] = x[n, 0, f] */
int spk_so3_put_l0(const float* src, const float* v, int64_t n_atoms, int lmax, int F, float* out, spk_stream_t stream);
int spk_so3_take_l0(const float* x, int64_t n_atoms, int lmax, int F, float* q, spk_stream_t stream);

/* ---- per-step model properties of DeviceMD (md/calculators/base_calculator.py:113-141) -------------------------------
 * dst[i] = src[i] * conversion.  Time series: counter (int64[2], device) = (steps completed, records stored); step
 * s = counter[0] + 1 is recorded when s % every == 0: buf[counter[1] * n + i] = src[i] (nothing once counter[1] reaches
 * capacity).  spk_md_record_advance then advances both counters; call it once per step after every spk_md_record. */
int spk_md_property(const float* src, int64_t n, float conversion, float* dst, spk_stream_t stream);
int spk_md_record(const float* src, int64_t n, const int64_t* counter, int64_t every, int64_t capacity, float* buf,
                  spk_stream_t stream);
int spk_md_record_advance(int64_t* counter, int64_t every, int64_t capacity, spk_stream_t stream);
/* velocity record (the FileLogger's MoleculeStream with store_velocities): on a recorded step (as spk_md_record)
 * buf[counter[1] * 3 n_atoms + 3 a + k] = momenta[a, k] / masses[a]; call it before spk_md_record_advance. */
int spk_md_record_velocities(const float* momenta, const float* masses, int64_t n_atoms, const int64_t* counter,
                             int64_t every, int64_t capacity, float* buf, spk_stream_t stream);

/* ---- gated equivariant output heads (csrc/equivariant.cu) -------------------------------------------------------------
 * nn/equivariant.py:57-71 (GatedEquivariantBlock), atomistic/atomwise.py:172-213 (DipoleMoment), :267-293
 * (Polarizability).  Vectors are [N, 3, F]; VW = mix_vectors(V) is [N, 3, 2Fo] with V = VW[..., :Fo], W = VW[..., Fo:].
 *
 * Hidden-block glue (the three Dense layers run on spk_dense_tc / spk_dense):
 *   ctx = [s | ||V||] [N, Fi+Fo] (no epsilon);  reverse: g_s = g_ctx[:, :Fi], g_VW[V columns] = g_ctx[:, Fi:] V / ||V||
 *   (0 where ||V|| = 0; the W columns are left to spk_geq_gate_bwd)
 *   s_out = act(x[:, :Fo]), v_out = x[:, Fo:] * W;  reverse: g_x [N, 2Fo], g_VW[W columns]  (g_s / g_v may be NULL) */
int spk_geq_ctx(const float* s, const float* VW, int64_t n_atoms, int Fi, int Fo, float* ctx, spk_stream_t stream);
int spk_geq_ctx_bwd(const float* g_ctx, const float* VW, int64_t n_atoms, int Fi, int Fo, float* g_s, float* g_VW,
                    spk_stream_t stream);
int spk_geq_gate(const float* x, const float* VW, int64_t n_atoms, int Fo, int act, float* s_out, float* v_out,
                 spk_stream_t stream);
int spk_geq_gate_bwd(const float* g_s, const float* g_v, const float* x, const float* VW, int64_t n_atoms, int Fo,
                     int act, float* g_x, float* g_VW, spk_stream_t stream);

#define SPK_HEAD_DIPOLE 0
#define SPK_HEAD_POLAR 1
/* weights of the last block (n_sout = n_vout = 1): Fi inputs, H gating hidden units (both <= 256) */
typedef struct {
    const float* wmix; /* [2, Fi]    mix_vectors.weight     */
    const float* w0;   /* [H, Fi+1]  scalar_net.0.weight    */
    const float* w0t;  /* [Fi+1, H]  its transpose          */
    const float* b0;   /* [H]                               */
    const float* w1;   /* [2, H]     scalar_net.1.weight    */
    const float* b1;   /* [2]                               */
    int32_t Fi, H, act, reserved;
} spk_head_tail_t;
size_t spk_head_workspace_bytes(int64_t n_atoms, int64_t n_sys);
/* Per-system head outputs.  With `tail` the last block runs per atom on (s [N,Fi], V [N,3,Fi]); without it (scalar
 * DipoleMoment) the charges q [N] are given.  Atoms of system m are [sys_ptr[m], sys_ptr[m+1]) (idx_m sorted).
 *   dipole:  q' = q + c_m, c_m = correct ? (Q_m - sum_m q) / n_m : 0 (0 for an empty system, Q = total_charge or 0),
 *            y_m = sum q' R + sum mu_atomic;  out [B, 3], or |y_m| [B] with `magnitude`
 *   polar:   out [B, 3, 3] = sum alpha I + sum (nu (x) R + R (x) nu)
 * Sums in fp64 through a fixed-shape segmented reduction: bitwise reproducible, no atomics.  q_atom [N] (may be NULL)
 * receives the tail's charges; saved [B, 8] fp64 keeps (c, mean R, y, n) of the dipole for spk_head_charges and the
 * reverse (zeros for the polarizability, whose reverse needs none of them). */
int spk_head_fwd(int kind, const spk_head_tail_t* tail, const float* s, const float* V, const float* q, const float* R,
                 const int64_t* idx_m, const int32_t* sys_ptr, const float* total_charge, int64_t n_atoms, int64_t n_sys,
                 int correct, int magnitude, float* out, float* q_atom, double* saved, void* workspace,
                 size_t workspace_bytes, spk_stream_t stream);
/* charges[i] = q_atom[i] + c_{m(i)} */
int spk_head_charges(const float* q_atom, const int64_t* idx_m, const double* saved, int64_t n_atoms, float* charges,
                     spk_stream_t stream);
/* Reverse of the tail head for g_out (the shape of out): g_s [N,Fi], g_V [N,3,Fi], g_R [N,3] (the direct position term) */
int spk_head_bwd(int kind, const spk_head_tail_t* tail, const float* s, const float* V, const float* R,
                 const int64_t* idx_m, const double* saved, const float* g_out, int64_t n_atoms, int correct,
                 int magnitude, float* g_s, float* g_V, float* g_R, spk_stream_t stream);
/* Reverse of the scalar dipole: g_hid[i, :] = g_q_i w1 (w1 [H] = the last Dense H -> 1) and g_R [N,3] */
int spk_head_scalar_bwd(const float* q, const float* R, const int64_t* idx_m, const double* saved, const float* g_out,
                        int correct, int magnitude, const float* w1, int64_t n_atoms, int H, float* g_hid, float* g_R,
                        spk_stream_t stream);
/* Reverse of spk_head_charges for the charge gradient g_charges [N]: g_q [N] = g_charges - mean_m(g_charges) with
 * `correct` (the per-system mean as an fp64 segmented sum, bitwise reproducible, no atomics), else g_charges. */
size_t spk_head_charges_bwd_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_head_charges_bwd(const float* g_charges, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                         int64_t n_sys, int correct, float* g_q, void* workspace, size_t workspace_bytes,
                         spk_stream_t stream);
/* spk_head_bwd / spk_head_scalar_bwd with the gradient g_q [N] of the tail's charges (from spk_head_charges_bwd) added
 * to the one the dipole sends to them; kind = SPK_HEAD_DIPOLE only. */
int spk_head_bwd_q(int kind, const spk_head_tail_t* tail, const float* s, const float* V, const float* R,
                   const int64_t* idx_m, const double* saved, const float* g_out, const float* g_q, int64_t n_atoms,
                   int correct, int magnitude, float* g_s, float* g_V, float* g_R, spk_stream_t stream);
int spk_head_scalar_bwd_q(const float* q, const float* R, const int64_t* idx_m, const double* saved, const float* g_out,
                          const float* g_q, int correct, int magnitude, const float* w1, int64_t n_atoms, int H,
                          float* g_hid, float* g_R, spk_stream_t stream);

/* ---- pair energies (csrc/pair_energy.cu; atomistic/nuclear_repulsion.py:81-104, atomistic/electrostatic.py:14-152) ---
 * Per edge e = (i, j), d = |r_ij| (an edge with d > d_max when d_max > 0 contributes nothing):
 *   ZBL:     a_k = Z_k^softplus(a_pow), a_ij = (a_i + a_j) softplus(a_div), c = normalize_L1(softplus(coefficients)),
 *            e = Z_i Z_j / d sum_k c_k exp(-a_ij softplus(exponents_k) d), times the cosine cutoff if cutoff > 0
 *   Coulomb: e = q_i q_j V(d), V = 1/d or (damped) f_sw / sqrt(d^2 + 1) + (1 - f_sw) / d with the switch function of
 *            (switch_on, switch_off); with cutoff > 0, V + shift^2 / V - 2 shift for d <= cutoff and 0 beyond
 *   Ewald real space (electrostatic.py:266-308): e = q_i q_j erfc(sqrt(alpha) d) / d, times 1 - f_sw(d) when
 *            switch_off != switch_on (the SwitchFunction screen); no cutoff, so padded lists need d_max
 * The ZBL parameters are read raw from device memory (softplus and normalisation on the device). */
#define SPK_PAIR_ZBL 0
#define SPK_PAIR_COULOMB 1
#define SPK_PAIR_DAMPED_COULOMB 2
#define SPK_PAIR_EWALD_REAL 3
#define SPK_PAIR_MAX_TERMS 16
typedef struct {
    int32_t kind;
    int32_t n_terms;           /* ZBL: number of screening terms (length of coefficients / exponents) */
    const float* a_pow;        /* ZBL: [1] */
    const float* a_div;        /* ZBL: [1] */
    const float* coefficients; /* ZBL: [n_terms] */
    const float* exponents;    /* ZBL: [n_terms] */
    double ke;
    double cutoff;             /* ZBL: cosine cutoff radius; Coulomb: shift cutoff; <= 0: none */
    double shift;              /* Coulomb with cutoff: V(cutoff) */
    double switch_on, switch_off;
    double d_max;              /* distance mask d <= d_max; <= 0: none */
    double alpha;              /* Ewald real space: the splitting parameter alpha (the square of the usual one) */
} spk_pair_t;
size_t spk_pair_energy_workspace_bytes(int64_t n_edges, int64_t n_sys);
/* energy [B] = 0.5 ke sum_{e in m} e_ij over the receiver slots [rowptr[sys_ptr[m]], rowptr[sys_ptr[m+1]]), summed in fp64
 * by the segmented-partial pass (bitwise reproducible, no atomics).  Z [N] for ZBL, q [N] for Coulomb. */
int spk_pair_energy_fwd(const spk_pair_t* p, const float* r_ij, const int64_t* idx_i, const int64_t* idx_j,
                        const int64_t* Z, const float* q, const int64_t* idx_m, const int32_t* rowptr,
                        const int32_t* slot_eid, const int32_t* sys_ptr, int64_t n_edges, int64_t n_sys, float* energy,
                        void* workspace, size_t workspace_bytes, spk_stream_t stream);
/* Reverse for g_E [B]: g_rij [E,3] = 0.5 ke g_E[m(e)] de/dd r_ij / d in edge order; for Coulomb and g_q != NULL also
 * g_q [N] = 0.5 ke g_E[m(a)] (sum over the receiver slots of a of q_j V + sum over its sender slots of q_i V) in the fixed
 * order of the two graph views. */
int spk_pair_energy_bwd(const spk_pair_t* p, const float* r_ij, const int64_t* idx_i, const int64_t* idx_j,
                        const int64_t* Z, const float* q, const int64_t* idx_m, const float* g_E, const int32_t* rowptr,
                        const int32_t* slot_j, const int32_t* slot_eid, const int32_t* sptr, const int32_t* pos_slot,
                        const int32_t* pos_i, int64_t n_atoms, int64_t n_edges, float* g_rij, float* g_q,
                        spk_stream_t stream);

/* ---- Ewald reciprocal and self terms (csrc/ewald.cu; atomistic/electrostatic.py:310-375) ---------------------------
 * Per system m with cell h [3,3] (rows = lattice vectors; fp32 in, fp64 inside), H = h^-1, V = |det h|, the integer
 * triples n [K,3] (fp32, the reference's kvecs buffer) and k = 2 pi n H^T:
 *   E_rec[m]  = ke (2 pi / V) sum_k f_k |S_k|^2,  f_k = exp(-k^2 / (4 alpha)) / k^2,  S_k = sum_{i in m} q_i e^{i k.r_i}
 *   E_self[m] = ke sqrt(alpha / pi) sum_{i in m} q_i^2
 *   energy[m] = addend[m] + E_rec[m] - E_self[m]      (addend: the real-space energy, or NULL)
 * The phases are 2 pi n.s_i with the fractional coordinates s_i = r_i H reduced mod 1 in fp64 (exact for integer n, so
 * unwrapped positions lose nothing).  Every sum runs in fp64 in a fixed order, without atomics: bitwise reproducible.
 * A system of zero volume gets NaN; an empty system gets addend[m].  Systems are the atom ranges [sys_ptr[m],
 * sys_ptr[m+1]) of spk_segment_ptr (idx_m sorted), n_sys <= 65535.  The launch shapes depend on n_atoms, n_sys and K
 * only.
 * workspace: spk_ewald_workspace_bytes(n_atoms, n_sys, K) bytes, 8-byte aligned; the forward leaves there what the
 * reverse reads, so the reverse takes the same workspace, untouched in between, with the same inputs. */
size_t spk_ewald_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n_k);
int spk_ewald_fwd(const float* R, const float* q, const float* cell, const float* kvecs, const int64_t* idx_m,
                  const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int64_t n_k, double ke, double alpha,
                  const float* addend, float* energy, void* workspace, size_t workspace_bytes, spk_stream_t stream);
/* Reverse for g_E [n_sys] (each output optional, NULL skips it):
 *   g_R [N,3]      = ke (2 pi / V) g_E sum_k 2 f_k q_i k (Im S_k cos t_ik - Re S_k sin t_ik),  t_ik = k.r_i
 *   g_q [N]       (+)= ke g_E [(2 pi / V) sum_k 2 f_k (Re S_k cos t_ik + Im S_k sin t_ik) - 2 sqrt(alpha / pi) q_i]
 *                   (accumulate_q: added to what g_q holds, e.g. the real-space charge gradient)
 *   g_cell [B,3,3] = -H^T [sum_i r_i (x) g_R_i - 2 g_E T + g_E E_rec I],  T = sum_k E_k (1/k^2 + 1/(4 alpha)) k (x) k
 *   virial [B,3,3] (+)= -g_E (E_rec I - 2 T), fp64, the strain derivative in the convention of spk_pairwise_virial
 *                   (accumulate_virial: added to what it holds) */
int spk_ewald_bwd(const float* R, const float* q, const float* cell, const float* kvecs, const int64_t* idx_m,
                  const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int64_t n_k, double ke, double alpha,
                  const float* g_E, float* g_R, float* g_q, int accumulate_q, float* g_cell, double* virial,
                  int accumulate_virial, void* workspace, size_t workspace_bytes, spk_stream_t stream);
/* ---- Smooth particle-mesh Ewald, reciprocal and self terms (csrc/pme.cu; Essmann et al., J. Chem. Phys. 103, 8577) --
 * Per system m with cell h [3,3] (fp32 in, fp64 inside), H = h^-1, V = |det h|, one mesh of n1 x n2 x n3 points for every
 * system and cardinal B-splines M_p of order p in {4, 6, 8}, with p <= n_a on every axis (an atom's p support points
 * along an axis are then distinct mesh points):
 *   Q_m(x)    = sum_{i in m} q_i prod_a M_p(n_a s_ia - x_a mod n_a),  s_i = r_i H reduced mod 1 in fp64
 *   E_rec[m]  = sum_{j != 0} theta_j |Q^_m(j)|^2,  theta_j = ke (2 pi / V) f_k |b(j)|^2,  f_k = exp(-k^2 / (4 alpha)) / k^2
 *   energy[m] = addend[m] + E_rec[m] - ke sqrt(alpha / pi) sum_{i in m} q_i^2
 * over the signed mesh frequencies j (a Nyquist index n_a / 2 of an even axis is left out), k = 2 pi H j and the Euler
 * spline moduli |b|^2.  The FFTs are the caller's, between the calls: spectrum = rfftn(mesh) over the three mesh axes
 * ([n_sys, n1, n2, n3 / 2 + 1] complex fp64, re/im interleaved) and potential = irfftn(conv) (fp64 [n_sys, n1, n2, n3]).
 * Every sum runs in fp64 in a fixed order without floating-point atomics: bitwise reproducible.  A system of zero volume
 * gets NaN; systems are the atom ranges of spk_segment_ptr, n_sys <= 65535, n_sys n1 n2 (n3 / 2 + 1) < 2^31.  The
 * launch shapes depend on n_atoms, n_sys and the mesh only.
 * workspace: spk_pme_workspace_bytes(...) bytes (0 for an invalid order or mesh), 8-byte aligned; spk_pme_spread leaves
 * there what spk_pme_energy and spk_pme_bwd read, so all three take the same workspace, untouched in between. */
size_t spk_pme_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n1, int64_t n2, int64_t n3, int order);
/* mesh [n_sys, n1, n2, n3] (fp64) = Q_m: bins the atoms by mesh brick and spreads their charges, every mesh point written
 * once */
int spk_pme_spread(const float* R, const float* q, const float* cell, const int64_t* idx_m, const int32_t* sys_ptr,
                   int64_t n_atoms, int64_t n_sys, int64_t n1, int64_t n2, int64_t n3, int order, double* mesh,
                   void* workspace, size_t workspace_bytes, spk_stream_t stream);
/* energy [n_sys] from spectrum = rfftn(mesh); conv (the spectrum's shape) = 2 n1 n2 n3 theta spectrum, whose irfftn is
 * the potential mesh dE_rec/dQ the reverse reads */
int spk_pme_energy(const float* q, const int32_t* sys_ptr, const double* spectrum, int64_t n_atoms, int64_t n_sys,
                   int64_t n1, int64_t n2, int64_t n3, int order, double ke, double alpha, const float* addend,
                   float* energy, double* conv, void* workspace, size_t workspace_bytes, spk_stream_t stream);
/* Reverse for g_E [n_sys] from potential = irfftn(conv) (each output optional, NULL skips it), with phi_i and grad phi_i
 * gathered over the p^3 support of atom i:
 *   g_R [N,3]      = g_E q_i H grad_s phi_i
 *   g_q [N]       (+)= g_E (phi_i - 2 ke sqrt(alpha / pi) q_i)          (accumulate_q as in spk_ewald_bwd)
 *   g_cell [B,3,3] = -H^T [sum_i r_i (x) g_R_i - 2 g_E T + g_E E_rec I],  T = sum_j E_j (1/k^2 + 1/(4 alpha)) k (x) k
 *   virial [B,3,3] (+)= -g_E (E_rec I - 2 T), fp64                        (accumulate_virial as in spk_ewald_bwd) */
int spk_pme_bwd(const float* R, const float* q, const int64_t* idx_m, const int32_t* sys_ptr, const double* potential,
                int64_t n_atoms, int64_t n_sys, int64_t n1, int64_t n2, int64_t n3, int order, double ke, double alpha,
                const float* g_E, float* g_R, float* g_q, int accumulate_q, float* g_cell, double* virial,
                int accumulate_virial, void* workspace, size_t workspace_bytes, spk_stream_t stream);
/* spk_pairwise_virial that adds W to what virial holds instead of overwriting it (the reciprocal Ewald virial is
 * deposited there first) */
int spk_pairwise_virial_add(const float* g_rij, const float* r_ij, const int32_t* rowptr, const int32_t* slot_eid,
                            const int32_t* sys_ptr, int64_t n_edges, int64_t n_sys, double* virial, void* workspace,
                            size_t workspace_bytes, spk_stream_t stream);

/* ---- batchwise L-BFGS relaxation (csrc/relax.cu; interfaces/batchwise_optimization.py:613-917) ----------------------
 * One optimizer per system (atoms [sys_ptr[m], sys_ptr[m+1])), state fp64 on the device, positions in optimizer units
 * (model positions x position_conversion).  order [n_sys] lists the systems of at most SPK_RELAX_WARP_ATOMS atoms first
 * (n_warp of them, one warp each), then the larger ones (one thread-block cluster each).  counter (int64[2]) = (steps
 * taken as the next step reads it, steps taken as the last step wrote it); spk_relax_converged must run between two
 * steps, on the forces the next step uses.
 *
 * spk_relax_step, with f = forces x force_conversion (0 on fixed atoms) and it = counter[0]:
 *   if it > 0: slot (it-1) % memory of s / y [memory, 3N] = r - r0, f0 - f; rho [memory, n_sys] = 1 / (y.s) if
 *              y.s > 1e-8, else 1;
 *   two-loop recursion over the last min(memory, it) entries with H0 = h0; p = 0 for a converged system;
 *   per system, p *= maxstep / longest if the longest per-atom step >= maxstep;
 *   r0 = r, f0 = f, r += damping p, model_positions = float(r / position_conversion), counter[1] = it + 1.
 * spk_relax_converged: fmax_sys[m] = max_a |f_a|, converged[m] = fmax_sys[m]^2 < fmax[0]^2, steps[m] = the counter[1]
 *   at which the system became converged (kept while it stays converged, -1 otherwise), n_unconverged[0] = count of
 *   unconverged systems, counter[0] = counter[1].
 * All sums run in a fixed order (bitwise reproducible), without atomics. */
#define SPK_RELAX_WARP_ATOMS 256
#define SPK_RELAX_MAX_MEMORY 4096
typedef struct {
    double* r;                 /* [N, 3] */
    double* r0;                /* [N, 3] */
    double* f0;                /* [N, 3] */
    double* s;                 /* [memory, N, 3] */
    double* y;                 /* [memory, N, 3] */
    double* rho;               /* [memory, n_sys] */
    double* p;                 /* [N, 3] step direction after masking and capping */
    int64_t* counter;          /* [2] */
    const double* fmax;        /* [1] convergence threshold */
    double* fmax_sys;          /* [n_sys] */
    int32_t* converged;        /* [n_sys] */
    int64_t* steps;            /* [n_sys] */
    int32_t* n_unconverged;    /* [1] */
    const uint8_t* fixed;      /* [N] or NULL */
    float* model_positions;    /* [N, 3] */
    const int32_t* sys_ptr;    /* [n_sys + 1] */
    const int32_t* order;      /* [n_sys] */
    int64_t n_atoms, n_sys, n_warp, memory;
    double force_conversion, position_conversion, maxstep, damping, h0;
} spk_lbfgs_t;
int spk_relax_step(const spk_lbfgs_t* state, const float* forces, spk_stream_t stream);
int spk_relax_converged(const spk_lbfgs_t* state, const float* forces, spk_stream_t stream);

/* ---- batchwise FIRE relaxation with an optional unit-cell filter (csrc/fire.cu; ASE's FIRE without downhill_check and
 * ASE's UnitCellFilter) ---------------------------------------------------------------------------------------------
 * One optimizer per system (atoms [sys_ptr[m], sys_ptr[m+1]), idx_m sorted), state fp64 on the device, in optimizer
 * units (model positions / cells x position_conversion, model energies x energy_conversion).  The generalized
 * coordinates of system m are the rows s [N, 3] of its atoms and, with filter = 1, the 9 values h[m] = cell_factor[m] F
 * (row-major), F the deformation gradient with cell = cell0 F^T (rows = lattice vectors); without a filter F = I and
 * s are the positions.  counter (int64[2]) = (steps taken as the next step reads it, steps taken as the last step wrote
 * it).  spk_fire_forces must run between two steps, on the forces (and virial) of the current positions.
 *
 * spk_fire_forces, with f = forces x force_conversion (0 on fixed atoms) and F = h / cell_factor:
 *   g [N, 3] = f_i F; with the filter hg [n_sys, 9] = P(Vir F^-T) / cell_factor, Vir = -(energy_conversion sym(W) +
 *   scalar_pressure V I), W = virial [n_sys, 3, 3] (fp64, model units, the strain derivative of spk_pairwise_virial),
 *   V = |det cell|, P the projections in ASE's order: hydrostatic_strain (tr / 3 I), the element-wise mask [9],
 *   constant_volume (tr / 3 off the diagonal);
 *   sums [n_sys, 3] = (v.g, v.v, g.g) over all generalized coordinates (fixed-order CTA partials, no atomics);
 *   fmax_sys[m] = sqrt(max_row |g_row|^2), converged[m] = fmax_sys^2 < fmax[0]^2, steps[m] = the counter[1] at which
 *   the system became converged (kept while it stays converged, -1 otherwise), n_unconverged[0], counter[0] = counter[1].
 * spk_fire_step, per unconverged system (a converged one keeps all its state): if started, ASE's mixing when v.g > 0
 *   (v = (1 - a) v + a g / |g| |v|; dt = min(dt finc, dtmax) and a *= fa if nsteps > nmin; nsteps += 1), else the
 *   reset (v = 0, a = astart, dt *= fdec, nsteps = 0); then v += dt g, dr = dt v, dr *= maxstep / |dr| if |dr| >
 *   maxstep (|dr| over all the system's coordinates, from the three sums); s += dr, h += dr, r = s F^T,
 *   model_positions = float(r / position_conversion), model_cell = float(cell0 F^T / position_conversion);
 *   counter[1] = counter[0] + 1.
 * workspace: spk_fire_workspace_bytes(n_atoms, n_sys) bytes, 8-byte aligned, untouched between the two calls. */
typedef struct {
    double* s;                 /* [N, 3] generalized atom coordinates */
    double* r;                 /* [N, 3] positions (may alias s without a filter) */
    double* v;                 /* [N, 3] */
    double* g;                 /* [N, 3] */
    double* h;                 /* [n_sys, 9] cell_factor F (filter only) */
    double* hv;                /* [n_sys, 9] (filter only) */
    double* hg;                /* [n_sys, 9] (filter only) */
    const double* cell0;       /* [n_sys, 9] the starting cell (filter only) */
    const double* cell_factor; /* [n_sys] (filter only) */
    double* dt;                /* [n_sys] */
    double* a;                 /* [n_sys] */
    int64_t* nsteps;           /* [n_sys] */
    int32_t* started;          /* [n_sys] 0 until the system's first step */
    double* sums;              /* [n_sys, 3] */
    double* coef;              /* [n_sys, 7] step coefficients, written and read by spk_fire_step */
    double* workspace;
    int64_t* counter;          /* [2] */
    const double* fmax;        /* [1] convergence threshold */
    double* fmax_sys;          /* [n_sys] */
    int32_t* converged;        /* [n_sys] */
    int64_t* steps;            /* [n_sys] */
    int32_t* n_unconverged;    /* [1] */
    const uint8_t* fixed;      /* [N] or NULL */
    float* model_positions;    /* [N, 3] */
    float* model_cell;         /* [n_sys, 3, 3] (filter only) */
    const int64_t* idx_m;      /* [N] */
    const int32_t* sys_ptr;    /* [n_sys + 1] */
    double mask[9];            /* element-wise mask of the cell forces (ones: no mask) */
    int64_t n_atoms, n_sys, nmin;
    int32_t filter, hydrostatic_strain, constant_volume, reserved;
    double force_conversion, energy_conversion, position_conversion, scalar_pressure;
    double maxstep, dtmax, finc, fdec, astart, fa;
} spk_fire_t;
size_t spk_fire_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_fire_forces(const spk_fire_t* state, const float* forces, const double* virial, spk_stream_t stream);
int spk_fire_step(const spk_fire_t* state, spk_stream_t stream);

/* ---- climbing-image nudged elastic band forces (csrc/neb.cu; Henkelman & Jonsson, J. Chem. Phys. 113, 9978 (2000);
 * Henkelman, Uberuaga & Jonsson, J. Chem. Phys. 113, 9901 (2000)) ---------------------------------------------------
 * A band is images 0 .. n+1 of the same atoms in the same order; images 0 and n+1 are fixed endpoints, the n =
 * n_images interior images move.  The batch holds the interior images of n_bands bands, band-major, image-major: band b
 * owns atoms [band_ptr[b], band_ptr[b+1]) = n images of A_b = (band_ptr[b+1] - band_ptr[b]) / n atoms, interior image
 * img = b n + i (i = 0 .. n-1 is image i+1 of the band) owns atoms [img_ptr[img], img_ptr[img+1]), idx_img [N] its
 * image per atom.  Endpoint rows: atom k of band b is row band_ptr[b] / n + k of r_initial / r_final [sum_b A_b, 3].
 * Everything is in optimizer units: positions (model x position_conversion), V = energies x energy_conversion,
 * F = forces x force_conversion, 0 on fixed atoms; end_energies [n_bands, 2] = (V_0, V_n+1) already in those units.
 *
 * spk_neb_forces, per interior image with D+ = R_{i+1} - R_i, D- = R_i - R_{i-1} over its 3 A_b coordinates (plain
 *   differences, never wrapped):
 *   sums a = D+.D+, b = D-.D-, c = D+.D-, d = F.D+, e = F.D- (fixed-order CTA partials, no atomics);
 *   tau = alpha D+ + beta D-: (1, 0) if V_{i+1} > V_i > V_{i-1}, (0, 1) if V_{i+1} < V_i < V_{i-1}, else with dV_max /
 *   dV_min the larger / smaller of |V_{i+-1} - V_i|: (dV_max, dV_min) if V_{i+1} > V_{i-1}, else (dV_min, dV_max); if
 *   that gives |tau| = 0 (a flat stretch), the bisector (1 / |D+|, 1 / |D-|) (a zero difference gives a zero weight);
 *   |tau|^2 = alpha^2 a + 2 alpha beta c + beta^2 b, F.tau = alpha d + beta e;
 *   the climbing image of a band, when climb[0] != 0: the interior image of the highest V, ties to the lowest index;
 *   gamma = -2 F.tau / |tau|^2 for the climbing image, else -F.tau / |tau|^2 + k (|D+| - |D-|) / |tau|; 0 if |tau| = 0;
 *   neb_forces [N, 3] fp32 = F + gamma tau, 0 on fixed atoms (F - (F.t) t + k (|D+| - |D-|) t with t = tau / |tau|,
 *   or F - 2 (F.t) t for the climbing image);
 *   coef [n_img, 3] = (alpha, beta, gamma); diag [n_img, 6] = (|tau|, F.t, the spring term k (|D+| - |D-|) (0 for the
 *   climbing image), |D+|, |D-|, 1 for the climbing image else 0); climbing [n_bands] = the climbing image's interior
 *   index i, -1 when climb[0] == 0.
 * climb is read on the device, so a captured call follows it.  The NEB forces drive spk_fire_step with the band as the
 * system (force_conversion = 1), whose |dr| cap and fmax test then run over every moving coordinate of the band.
 * Three launches; workspace: spk_neb_workspace_bytes(n_atoms, n_img) bytes, 8-byte aligned. */
typedef struct {
    const double* r;            /* [N, 3] interior positions (FIRE's r) */
    const double* r_initial;    /* [sum_b A_b, 3] image 0 of every band */
    const double* r_final;      /* [sum_b A_b, 3] image n+1 of every band */
    const double* end_energies; /* [n_bands, 2] */
    const int32_t* climb;       /* [1] 0: plain NEB, else climbing image */
    const uint8_t* fixed;       /* [N] or NULL */
    const int64_t* idx_img;     /* [N] */
    const int32_t* img_ptr;     /* [n_img + 1] */
    const int32_t* band_ptr;    /* [n_bands + 1] */
    double* coef;               /* [n_img, 3] */
    double* diag;               /* [n_img, 6] */
    int32_t* climbing;          /* [n_bands] */
    float* neb_forces;          /* [N, 3] */
    double* workspace;
    int64_t n_atoms, n_images, n_bands;
    double k, force_conversion, energy_conversion;
} spk_neb_t;
size_t spk_neb_workspace_bytes(int64_t n_atoms, int64_t n_images);
int spk_neb_forces(const spk_neb_t* state, const float* forces, const float* energies, spk_stream_t stream);

/* ---- model ensembles (csrc/ensemble.cu; md/calculators/ensemble_calculator.py:38-59,
 * interfaces/batchwise_optimization.py:36-72, interfaces/ase_interface.py:340-432) ------------------------------------
 * The K members' outputs are stacked fp32 slots [K, ...] (slot k = member k).  Every statistic runs in fp64 over k in
 * ascending order, in two passes (the mean, then the sum of squared deviations ss from it), without atomics: bitwise
 * reproducible.
 *
 * spk_ensemble_moments, element-wise over x [K, n]: mean = sum_k x / K, var = ss / (K - ddof) (ddof 0 or 1, K > ddof);
 *   mean_out = mean * mean_scale, var_out = var * spread_scale, std_out = sqrt(var) * spread_scale (each optional).
 * spk_ensemble_forces, one thread per atom of forces [K, N, 3] (K >= 2): mean [N, 3] = mean * mean_scale, var [N, 3] =
 *   the unbiased variance * spread_scale (each optional) and, with sys_terms, per system s (atoms [sys_ptr[s],
 *   sys_ptr[s+1]), idx_m sorted) sys_terms[s] = (sum_i ||sd_i||, sum_i ||sd_i|| / (||mu_i|| + 1e-8)) with sd_i the
 *   ddof-0 standard deviation and mu_i the mean of F_i * spread_scale; 0 for an empty system.  workspace:
 *   spk_ensemble_workspace_bytes(N, n_sys) bytes, 8-byte aligned (only with sys_terms).
 * spk_ensemble_uncertainty, one thread per system: out [n_sys] fp64 = w_e u_E + w_f u_F + w_s u_S, each term only if
 *   its weight is > 0.  u_E = std_0(E * energy_scale) of energy [K, n_sys] (relative: over |mean| + 1e-8); u_F =
 *   sys_terms[s][relative] / n_atoms(s), 0 for a system without atoms (the reference would take the mean of nothing);
 *   u_S = the mean over the 3 rows of ||std_0 of the row|| of stress [K, n_sys, 3, 3] * stress_scale (relative: each
 *   row over ||mean row|| + 1e-8).  out_f32 [n_sys] (optional, as out) receives the same values rounded to fp32. */
size_t spk_ensemble_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_ensemble_moments(const float* x, int64_t K, int64_t n, int ddof, double mean_scale, double spread_scale,
                         float* mean, float* var, float* std, spk_stream_t stream);
int spk_ensemble_forces(const float* forces, int64_t K, const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms,
                        int64_t n_sys, double mean_scale, double spread_scale, float* mean, float* var,
                        double* sys_terms, void* workspace, size_t workspace_bytes, spk_stream_t stream);
int spk_ensemble_uncertainty(const float* energy, double energy_scale, const double* force_sums, const int32_t* sys_ptr,
                             const float* stress, double stress_scale, int64_t K, int64_t n_sys, int relative,
                             double energy_weight, double force_weight, double stress_weight, double* out,
                             float* out_f32, spk_stream_t stream);

/* ---- vibrational analysis (csrc/vibrations.cu; ASE's Vibrations / Infrared, atomistic/response.py:95-431,
 * nn/utils.py:21-126) --------------------------------------------------------------------------------------------------
 * Finite-difference Hessians of a B-system batch (N atoms, system m = atoms [sys_ptr[m], sys_ptr[m+1]), n_m atoms,
 * coordinates d = 3 a + k) from C = n_cols * nfree replica-major copies: copy c = d_local * nfree + s holds atoms
 * [c N, (c+1) N) and systems [c B, (c+1) B) and displaces coordinate d = chunk * n_cols + d_local of every system by
 * (float)(o_s * delta), o = (-1, +1) for nfree 2 and (-2, -1, +1, +2) for nfree 4; systems with d >= 3 n_m stay
 * undisplaced in that copy (idle).  n_displaced (int64[B], optional) restricts the displaced coordinates of system m to
 * those of its first n_displaced[m] atoms, d < 3 n_displaced[m] (NULL: all n_m atoms).  counter (int64[2]) = (chunk the
 * next displacement reads, chunk the last displacement wrote + 1); zero it before the first chunk.
 *
 * spk_vib_displace: positions [C N, 3] = base with the displacement rounded to fp32 (__fadd_rn); steps [C, B] fp64 =
 *   (double)displaced - (double)base of the displaced coordinate (0 for idle copies); counter[1] = counter[0] + 1.
 * spk_vib_assemble, after the model wrote forces [C N, 3] (and dipole [C B, 3] / polar [C B, 3, 3]): for chunk =
 *   counter[1] - 1 and every non-idle (system, d): with w_s the weights of the derivative at 0 of the polynomial through
 *   (steps[c_s, m], y_s), h_raw[hess_ptr[m] + d 3 n_m + r] = -sum_s w_s forces_r (column d, stored transposed),
 *   for d < 3 n_displaced[m] (the block of system m then holds 9 n_displaced[m] n_m values),
 *   dipole_deriv [N, 3, 3] element [i, comp, dir] and polar_deriv [N, 3, 3, 3] element [i, a, b, dir] (each optional)
 *   = sum_s w_s y_s with atom i = sys_ptr[m] + d / 3, dir = d % 3; counter[0] = counter[1].
 * spk_vib_finish, once after the last chunk: H = (h_raw + h_raw^T) / 2 per system; hessian [sum n_m^2, 3, 3] fp64 in
 *   the Response layout (row i n_m + j, block [a, b] = H[3 i + a, 3 j + b]) at hess_ptr[m] (= 9 sum_{m' < m} n_m'^2) and
 *   hessian_mw [3 n_m, 3 n_m] at the same offset = H * mw_scale / sqrt(masses[i] masses[j]).  max_atoms = max_m n_m.
 *   Needs n_displaced == NULL.
 * No atomics; every value is written once: bitwise reproducible. */
typedef struct {
    const float* base;         /* [N, 3] undisplaced model positions */
    float* positions;          /* [C N, 3] replica positions */
    double* steps;             /* [C, B] realised steps */
    int64_t* counter;          /* [2] */
    const float* forces;       /* [C N, 3] */
    const float* dipole;       /* [C B, 3] or NULL */
    const float* polar;        /* [C B, 3, 3] or NULL */
    const int64_t* idx_m;      /* [N] */
    const int32_t* sys_ptr;    /* [B + 1] */
    const int64_t* n_displaced;   /* [B] displaced atoms per system (the first ones), or NULL: all */
    const int64_t* hess_ptr;   /* [B + 1] */
    const double* masses;      /* [N] */
    double* h_raw;             /* [sum 9 n_m^2], or [sum 9 n_displaced[m] n_m] */
    double* hessian;           /* [sum n_m^2, 3, 3] */
    double* hessian_mw;        /* [sum 9 n_m^2] */
    double* dipole_deriv;      /* [N, 3, 3] or NULL */
    double* polar_deriv;       /* [N, 3, 3, 3] or NULL */
    int64_t n_atoms, n_sys, n_cols, nfree, max_atoms;
    double delta;              /* step in model length units */
    double mw_scale;           /* energy_conversion / position_conversion^2 */
} spk_vib_t;
int spk_vib_displace(const spk_vib_t* params, spk_stream_t stream);
int spk_vib_assemble(const spk_vib_t* params, spk_stream_t stream);
int spk_vib_finish(const spk_vib_t* params, spk_stream_t stream);

/* ---- phonons of crystals (csrc/phonons.cu; the method of ASE's Phonons) ------------------------------------------------
 * System m (of B) has n_m primitive atoms [prim_ptr[m], prim_ptr[m+1]) and a supercell of L = n_cells primitive cells
 * (supercell matrix M, rows of the supercell = M . cell); supercell atom j = l n_m + b is primitive atom b translated by
 * lattice[l] (int32 [L, 3], lattice[0] = 0), and neg[l] is the index of -lattice[l] modulo the supercell.  Row
 * fc_ptr[m] + a n_m L + j (fc_ptr[m] = sum_{m' < m} n_m'^2 L, n_rows = fc_ptr[B]) holds the block Phi(a, 0; j) [3, 3].
 *
 * spk_ph_force_constants: h_raw = the finite differences of spk_vib_assemble with n_displaced[m] = n_m (per system rows
 *   d = 3 a + alpha of 3 n_m L columns, at 9 fc_ptr[m]) -> force_constants [n_rows, 3, 3] after `rounds` rounds of:
 *   Phi(a, 0; b, l) <- (Phi(a, 0; b, l) + Phi(b, 0; a, neg[l])^T) / 2, then, if acoustic, Phi(a, 0; a, 0) -= sum_j
 *   Phi(a, 0; j) (the sum in ascending j).  Without acoustic at most one round runs (a second one is the identity).
 *   work: [n_rows, 3, 3] scratch.  1 + rounds launches.
 * spk_ph_images: for every row, the supercell-lattice images of atom j closest to atom a (positions [N_prim, 3], cell
 *   [B, 3, 3] primitive rows, super_cell / super_inv [B, 3, 3] = M . cell and its inverse, heights [B, 3] = the
 *   supercell's plane spacings, all fp64): the images within tie_tol of the shortest distance; img_count[row] = their
 *   number (may exceed SPK_PH_MAX_IMAGES: then only the first SPK_PH_MAX_IMAGES are stored and the table is unusable),
 *   img_lattice [n_rows, SPK_PH_MAX_IMAGES, 3] = their primitive lattice translations.
 * spk_ph_dynmat: dyn [n_q, dyn_ptr[B]] complex128 (re, im), system m at dyn_ptr[m] (= 9 sum_{m' < m} n_m'^2) as
 *   [3 n_m, 3 n_m]: D_{a alpha, b beta}(q) = sum_l sum_images Phi(a, 0; l n_m + b)[alpha, beta] e^{2 pi i q . n_image}
 *   / img_count * mw_scale / sqrt(masses[a] masses[b]) for q [n_q, 3] in reduced reciprocal coordinates.  max_atoms =
 *   max_m n_m.
 * spk_ph_dos: out [B, n_grid] = sum_{q, k} exp(-(grid - freq[q, 3 prim_ptr[m] + k])^2 / (2 width^2)) / (width sqrt(2 pi)
 *   n_q) over the 3 n_m modes of system m; freq [n_q, n_modes], n_modes = 3 prim_ptr[B].  Fixed loop order (q, k).
 * spk_ph_thermo: per segment s = t B + m (items [seg_ptr[s], seg_ptr[s+1]) = the n_q 3 n_m modes of system m, n_items =
 *   seg_ptr[n_temps B]): out [n_temps B, 6] = per primitive cell, with e = freq ev_per_invcm, x = e / (k_b T):
 *   (sum e / 2, sum e / 2 + k_b T ln(1 - e^-x), k_b sum (x / (e^x - 1) - ln(1 - e^-x)), k_b sum (x / (2 sinh(x/2)))^2) / n_q
 *   over the modes with freq >= min_freq (T = 0: zero-point terms only), then the number of modes left out and of those
 *   with freq < 0.  Segmented fp64 sums of segscan.cuh (2 launches) in spk_ph_thermo_workspace_bytes(n_items, n_temps B)
 *   bytes of workspace.
 * No atomics; every value is written once: bitwise reproducible. */
#define SPK_PH_MAX_IMAGES 8
typedef struct {
    const double* h_raw;       /* [9 n_rows] finite differences (spk_vib_assemble) */
    double* force_constants;   /* [n_rows, 3, 3] */
    double* work;              /* [n_rows, 3, 3] */
    const int32_t* prim_ptr;   /* [B + 1] */
    const int64_t* fc_ptr;     /* [B + 1] */
    const int32_t* lattice;    /* [L, 3] */
    const int32_t* neg;        /* [L] */
    const double* positions;   /* [N_prim, 3] primitive positions */
    const double* cell;        /* [B, 3, 3] */
    const double* super_cell;  /* [B, 3, 3] */
    const double* super_inv;   /* [B, 3, 3] */
    const double* heights;     /* [B, 3] */
    const double* masses;      /* [N_prim] */
    int32_t* img_count;        /* [n_rows] */
    int32_t* img_lattice;      /* [n_rows, SPK_PH_MAX_IMAGES, 3] */
    int32_t supercell[9];      /* M, row-major */
    int64_t n_sys, n_prim, n_rows, n_cells, max_atoms, rounds;
    int32_t acoustic, reserved;
    double tie_tol;            /* model length units */
    double mw_scale;           /* energy_conversion / position_conversion^2 */
} spk_ph_t;
int spk_ph_force_constants(const spk_ph_t* params, spk_stream_t stream);
int spk_ph_images(const spk_ph_t* params, spk_stream_t stream);
int spk_ph_dynmat(const spk_ph_t* params, const double* q, int64_t n_q, const int64_t* dyn_ptr, void* dyn,
                  spk_stream_t stream);
int spk_ph_dos(const double* freq, int64_t n_q, int64_t n_modes, const int32_t* prim_ptr, int64_t n_sys,
               const double* grid, int64_t n_grid, double width, double* out, spk_stream_t stream);
size_t spk_ph_thermo_workspace_bytes(int64_t n_items, int64_t n_seg);
int spk_ph_thermo(const double* freq, int64_t n_q, int64_t n_modes, const int32_t* prim_ptr, int64_t n_sys,
                  const double* temperatures, int64_t n_temps, const int32_t* seg_ptr, int64_t n_items, double min_freq,
                  double ev_per_invcm, double k_b, double* out, void* workspace, size_t workspace_bytes,
                  spk_stream_t stream);

/* ---- vibrational spectra from recorded MD series (csrc/spectra.cu; md/data/spectra.py) ------------------------------
 * spk_spectrum_series: records [T, P, stride] fp32 (P replicas).  Output field f (of F) is
 *   x_f[t] = sum_{j<3, index[f, j] >= 0} coef[f, j] d(index[f, j], t),  d(i, t) = c(i, t) (derivative == 0, n = T) or
 *   (c(i, t + 2) - c(i, t)) / (2 dt_fs) (derivative != 0, n = T - 2),  c(i, t) = (sum_r records[t, r, i]) / P,
 *   all in fp64; then mean[f] = sum_t x_f / n, std[f] = sqrt(sum_t (x_f - mean)^2 / n) and z [F, n] = (x - mean) / std.
 *   index [F, 3] int64, coef [F, 3] fp64, mean / std [F] fp64 (device).  Fixed-order sums, no atomics.
 * spk_spectrum_autocorrelation: channel c holds the fields [ch_ptr[c], ch_ptr[c+1]) of z [F, n] with weights w [F]:
 *   acf [C, L] = (1/n) sum_f w_f sum_{t < n-k} z_f[t] z_f[t+k] for k < L (L <= n - 1), computed as the band of the Gram
 *   matrix on the fp64 tensor cores over fixed time chunks of SPK_SPECTRUM_CHUNK rows; the per-chunk partials (in the
 *   workspace) are summed in a fixed order, so a channel's result does not depend on the other channels of the launch.
 * spk_spectrum_transform: out [C, 4L] = 2 dt_fs |sum_{i<L} acf[c, i] window[i] cos(pi m (2i+1) / (8L))| (window NULL:
 *   none), the DCT-II form of |dt FFT| of the zero-padded, mirrored series; m (2i+1) is reduced modulo 16 L before the
 *   cosine, which comes from a quarter-wave table of cospi values.
 * Both take spk_spectrum_workspace_bytes(C, n, L) bytes of workspace, 8-byte aligned. */
#define SPK_SPECTRUM_CHUNK 2048
size_t spk_spectrum_workspace_bytes(int64_t n_channels, int64_t n, int64_t n_lags);
int spk_spectrum_series(const float* records, int64_t T, int64_t P, int64_t stride, const int64_t* index,
                        const double* coef, int64_t F, int derivative, double dt_fs, double* z, double* mean, double* std,
                        spk_stream_t stream);
int spk_spectrum_autocorrelation(const double* z, int64_t n, const int64_t* ch_ptr, const double* weight,
                                 int64_t n_channels, int64_t n_lags, double* acf, void* workspace,
                                 size_t workspace_bytes, spk_stream_t stream);
int spk_spectrum_transform(const double* acf, int64_t n_channels, int64_t n_lags, const double* window, double dt_fs,
                           double* out, void* workspace, size_t workspace_bytes, spk_stream_t stream);

/* ---- streaming autocorrelation of the live MD state (csrc/spectra.cu) -----------------------------------------------
 * A stream of F fields and L lags keeps, per field, y[t] = x[t] - x[0] and S[k] = sum_{t < n-k} y[t] y[t+k] (k < L),
 * Y = sum_t y[t], the first L values and a ring of the last L + SPK_SPECTRUM_STREAM_BLOCK values, all fp64, in one
 * zero-initialised buffer of spk_spectrum_stream_state_bytes(F, L) = 8 F (3 L + SPK_SPECTRUM_STREAM_BLOCK + 8) bytes
 * (2.43 GB, 0.81 GB per array, for the 24 576 velocity components of 8192 atoms at L = 4096; 76 MB for the 768 IR
 * fields of 256 molecules).
 * spk_spectrum_stream_push: on the steps with (counter[0] + 1) % every == 0 (the recorder's), frame
 *   r = counter[0] / every of field f is x_f as spk_spectrum_series forms it from a record, here read from the live
 *   state: component i of replica p is source[p stride + i] (fp32), divided by masses[(p stride + i) / 3] when masses
 *   is not NULL (velocities from momenta [P N, 3], stride = 3 N, as spk_md_record_velocities); derivative fields lag
 *   two frames.  After every SPK_SPECTRUM_STREAM_BLOCK samples the block's band products are added to S in a fixed order:
 *   the accumulators do not depend on how the steps are grouped into calls.  Two launches, no atomics,
 *   graph-capturable; counter is not advanced.
 * spk_spectrum_stream_finalise: after n samples (n - 1 >= n_out, n_out <= L), channel c of the fields
 *   fields[ch_ptr[c] .. ch_ptr[c+1]) with weights w: acf [C, n_out] = sum_i w_i C_i[k] with the normalised
 *   autocorrelation of field i, n var C[k] = S[k] - m (2 Y - H[k] - tail[k]) + (n - k) m^2, m = Y / n,
 *   var = S[0] / n - m^2, H[k] / tail[k] the sums of the first / last k values (the partial block is added to S on the
 *   fly; the state is not changed).  Workspace: spk_spectrum_stream_finalise_workspace_bytes(n_sel, n_out) =
 *   8 n_sel n_out bytes.  Two launches. */
#define SPK_SPECTRUM_STREAM_BLOCK 64
size_t spk_spectrum_stream_state_bytes(int64_t n_fields, int64_t n_lags);
size_t spk_spectrum_stream_finalise_workspace_bytes(int64_t n_fields, int64_t n_lags);
int spk_spectrum_stream_push(const float* source, const float* masses, int64_t P, int64_t stride, const int64_t* index,
                             const double* coef, int64_t F, int derivative, double dt_fs, const int64_t* counter,
                             int64_t every, int64_t n_lags, double* state, spk_stream_t stream);
int spk_spectrum_stream_finalise(const double* state, int64_t F, int64_t n_lags, int64_t n, const int64_t* fields,
                                 int64_t n_sel, const int64_t* ch_ptr, const double* weight, int64_t n_channels,
                                 int64_t n_out, double* acf, void* workspace, size_t workspace_bytes,
                                 spk_stream_t stream);

/* ---- set-up and steadying of the device MD state (csrc/system_motion.cu; md/system.py:258-315,652-684,
 * md/initial_conditions.py:50-188, md/simulation_hooks/basic_hooks.py:55-78) --------------------------------------------
 * Systems as for the thermostats: idx_m [n_atoms] int64 sorted, sys_ptr [n_sys+1] int32; positions / momenta [n_atoms,3]
 * fp32 in place, model_positions (nullable) = positions * position_conversion.  step (nullable) is a device int64 step
 * counter: with it, a call does nothing unless step[0] % every == 0 (hooks inside a captured step); it is not advanced.
 * spk_md_remove_motion: in the order of the flags' bits, per system, with all sums in fp64 and a fixed order (no atomics):
 *   SPK_MOTION_CENTER_OF_MASS  x -= sum m x / sum m;
 *   SPK_MOTION_TRANSLATION     p -= sum p / n_s (unweighted mean, system.py:278-283);
 *   SPK_MOTION_ROTATION        about the origin: I = sum m (|x|^2 1 - x x^T), L = sum x x p, w = I^+ L, p -= m (w x x),
 *                              with I^+ the pseudo-inverse that drops eigenvalues <= SPK_MOTION_PINV_RTOL x the largest
 *                              (single atoms, linear molecules, empty systems); I^-1 where I is regular.
 * spk_md_wrap_positions: positions [n_beads, n_atoms, 3] (n_beads = 1: classical); the centroid of the beads of atom a has
 *   fractional coordinates f = x_c C^-1 in the fp64 cell C = cell + idx_m[a] * cell_stride (rows = lattice vectors,
 *   cell_stride 0 = one cell for all systems, or 9); on the axes j with pbc[idx_m[a] * pbc_stride + j] != 0 (pbc_stride 0
 *   or 3) every bead moves by -floor(f_j + eps) C_j, so the centroid's f_j ends in [-eps, 1 - eps).  Every cell must have a
 *   non-zero volume.
 * spk_md_initial_momenta: p = w xi with w = m (uniform != 0) or sqrt(m kB temperature[idx_m]) (Maxwell-Boltzmann),
 *   xi ~ N(0,1) from Philox4x32-10 with key = seed and counter = (atom index, SPK_MOTION_DRAW_APPLICATION), normals 0..2
 *   for x, y, z as in spk_md_langevin, whose application counter never reaches that index.  uniform != 0 then rescales
 *   every system to its temperature exactly (the fixed-order sum of spk_md_kinetic_energy); a system at T = 0 keeps its p.
 *   temperature [n_sys] fp64 on the device.
 * spk_md_step_advance: step[0] += 1, once per step after the hooks.
 * Both per-system entry points take spk_md_motion_workspace_bytes(n_atoms, n_sys) bytes of workspace, 8-byte aligned. */
#define SPK_MOTION_CENTER_OF_MASS 1
#define SPK_MOTION_TRANSLATION 2
#define SPK_MOTION_ROTATION 4
#define SPK_MOTION_PINV_RTOL 1e-10
#define SPK_MOTION_DRAW_APPLICATION 0xFFFFFFFFFFFFFFFFull
size_t spk_md_motion_workspace_bytes(int64_t n_atoms, int64_t n_sys);
int spk_md_remove_motion(float* positions, float* model_positions, float* momenta, const float* masses,
                         const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_sys, int flags,
                         float position_conversion, const int64_t* step, int64_t every, void* workspace,
                         size_t workspace_bytes, spk_stream_t stream);
int spk_md_wrap_positions(float* positions, float* model_positions, const int64_t* idx_m, int64_t n_atoms,
                          int32_t n_beads, const double* cell, int64_t cell_stride, const uint8_t* pbc, int64_t pbc_stride,
                          double eps, float position_conversion, const int64_t* step, int64_t every, spk_stream_t stream);
int spk_md_initial_momenta(float* momenta, const float* masses, const int64_t* idx_m, const int32_t* sys_ptr,
                           int64_t n_atoms, int64_t n_sys, int uniform, double kB, const double* temperature, uint64_t seed,
                           void* workspace, size_t workspace_bytes, spk_stream_t stream);
int spk_md_step_advance(int64_t* step, spk_stream_t stream);

/* ---- structural observables of the device MD (csrc/structure.cu; DESIGN.md section 24) ------------------------------
 * Both entry points are hooks inside the captured step: with step (nullable, a device int64 step counter, not advanced)
 * every kernel returns at once unless step[0] % every == 0.  No float atomics; every fp64 sum has a fixed order.
 * spk_rdf_accumulate: the pairs the neighbour list lists at cutoff r_max (spk_neighbor_list: ordered (i, j, S) with
 *   |R_j - R_i + S cell| < r_max, (i, i, 0) excluded, self images included; R [n_atoms, 3], cell [n_sys, 9] fp32, pbc
 *   [n_sys, 3], all systems periodic) are binned by distance, bin floor(d n_bins / r_max), without being written out.
 *   Atom i of type ti = type[i] and j of type tj count in slot slot_of[ti n_types + tj] (-1: none) and in total_slot
 *   (-1: none), as integers.  Then acc [n_out, n_slots, n_bins] fp64 += sum_r V_s counts[s] over the systems
 *   s = r n_out + o (r ascending; n_out divides n_sys: the beads of a ring polymer fold onto their system),
 *   volume_sum [n_out] += sum_r V_s and frames[0] += 1, with V_s = |det(volume_cell + s volume_cell_stride)| x
 *   volume_scale (fp64, stride 0 or 9).  Workspace: spk_rdf_workspace_bytes(n_atoms, n_sys, n_slots, n_bins) bytes,
 *   zero-initialised once: its count region is left zero by every call.  Seven launches (sampling flag, grid setup,
 *   bin, sort, cell bounds, traversal, fold); only the sort does work on steps that do not sample.
 * spk_msd_accumulate: per atom a of n_atoms (ring polymers: the centroid of the n_beads copies positions[r n_atoms + a],
 *   replica-major) in systems idx_m / sys_ptr [n_sys + 1], species[a] in [0, n_species), n_species <= 8.  State, zero at
 *   the start: track [n_atoms, 6] fp64 (unwrapped position u, last sampled position), origins [n_slots, n_atoms, 3],
 *   origin_com [n_slots, n_sys, 3], acc [n_sys, n_species, n_lags] fp64, count [n_lags] int64, meta [2] int64 (samples
 *   taken, jump flag).  Sample n: u += x - last with the fractional components of the periodic axes wrapped to
 *   [-1/2, 1/2) in the cell of the atom's system (cell fp64 [*, 9] with stride 0 or 9, pbc [*, 3] with stride 0 or 3;
 *   both NULL for open systems); meta[1] = 1 if that displacement is longer than half the shortest periodic height.
 *   Every origin_every samples u (and, with remove_com, the mass-weighted centre of u per system) goes to origin slot
 *   (n / origin_every) % n_slots, n_slots = ceil(n_lags / origin_every); then for every held origin o with lag
 *   n - n_o < n_lags, acc[s, c, lag] += sum over the atoms of species c in s of |u - u_o - (com - com_o)|^2 and
 *   count[lag] += 1.  Workspace: spk_msd_workspace_bytes(n_atoms, n_sys, n_species, n_slots) = 8 (1 + 7 n_sys + 4 n_cta +
 *   n_slots + n_slots (n_sys + n_cta) W) bytes, n_cta = ceil(n_atoms / 256), W = n_species rounded up to 1, 2, 4 or 8.
 *   Seven launches with remove_com, five without. */
size_t spk_rdf_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n_slots, int64_t n_bins);
int spk_rdf_accumulate(const float* R, const float* cell, const uint8_t* pbc, const int32_t* sys_ptr, int64_t n_atoms,
                       int64_t n_sys, const int32_t* type, int64_t n_types, const int32_t* slot_of, int32_t total_slot,
                       int64_t n_slots, float r_max, int64_t n_bins, const double* volume_cell,
                       int64_t volume_cell_stride, double volume_scale, int64_t n_out, const int64_t* step,
                       int64_t every, double* acc, double* volume_sum, int64_t* frames, void* workspace,
                       size_t workspace_bytes, spk_stream_t stream);
size_t spk_msd_workspace_bytes(int64_t n_atoms, int64_t n_sys, int64_t n_species, int64_t n_slots);
int spk_msd_accumulate(const float* positions, int64_t n_atoms, int32_t n_beads, const float* masses,
                       const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_sys, const int32_t* species,
                       int64_t n_species, const double* cell, int64_t cell_stride, const uint8_t* pbc,
                       int64_t pbc_stride, int remove_com, int64_t n_lags, int64_t origin_every, int64_t n_slots,
                       const int64_t* step, int64_t every, double* track, double* origins, double* origin_com,
                       double* acc, int64_t* count, int64_t* meta, void* workspace, size_t workspace_bytes,
                       spk_stream_t stream);

/* ---- temperature replica exchange in the device MD (csrc/exchange.cu; DESIGN.md section 25) ------------------------
 * spk_remd_exchange: one exchange attempt over n_groups * n_rungs systems, rung-major (system k n_groups + g is rung k of
 *   group g; the systems of a group have equal atom counts, so atom a of system s sits at sys_ptr[s] + a).  With step
 *   (nullable, a device int64 step counter, not advanced) both kernels return at once unless step[0] % every == 0.
 *   Attempt n = attempt[0] (device int64, advanced by one) tries the pairs (k, k + 1) with k = n (mod 2) of every group:
 *   Delta = (1 / (kB T_k) - 1 / (kB T_k+1)) (U_k - U_k+1) in fp64 with U = energy[s] * energy_conversion and T =
 *   temperature[s] (fp64, K); the pair is accepted iff Delta >= 0 or u < exp(Delta), u = (x + 1/2) 2^-32 with x word 0
 *   of the Philox4x32-10 draw of key seed and counter (g (n_rungs - 1) + k, 2^63 + n).  decision [n_groups, n_rungs - 1]
 *   uint8 is set to 1 for the pairs that swap on this attempt and 0 for the others; attempted / accepted
 *   [n_groups, n_rungs - 1] int64 count the tried and accepted pairs; walker [n_rungs n_groups] int32 exchanges its two
 *   entries on every swap.  A swap exchanges the momenta [n_atoms, 3] of the two systems, rescaled by
 *   sqrt(T_new / T_old) in fp64 and rounded once to fp32, and the rows of every buffer of *buffers (nullable: none): per
 *   atom or per system, width floats each, copied unchanged.  No atomics.  Two launches (decide, swap). */
#define SPK_REMD_MAX_BUFFERS 16
typedef struct {
    int32_t n_buffers;     /* buffers used, <= SPK_REMD_MAX_BUFFERS */
    int32_t per_atom[16];  /* 1: one row per atom, 0: one row per system */
    int64_t width[16];     /* floats per row, >= 1 */
    float* data[16];       /* device fp32 buffers, swapped in place */
} spk_remd_buffers_t;

int spk_remd_exchange(const float* energy, double energy_conversion, const double* temperature, double kB,
                      const int64_t* idx_m, const int32_t* sys_ptr, int64_t n_atoms, int64_t n_groups, int32_t n_rungs,
                      uint64_t seed, const int64_t* step, int64_t every, int64_t* attempt, int32_t* walker,
                      int64_t* attempted, int64_t* accepted, uint8_t* decision, float* momenta,
                      const spk_remd_buffers_t* buffers, spk_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SPK_B200_H */

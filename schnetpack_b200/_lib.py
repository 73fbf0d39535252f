"""ctypes binding of the C-ABI library ``csrc/libspk_b200.so`` (declared in ``include/spk_b200.h``).

There is NO fallback: if the library is missing (not built) importing any op raises, and every op raises when it is
handed a non-CUDA tensor.  torch is used only as the owner of device memory and streams.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64, c_void_p
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SPK_B200_LIB") or os.path.join(HERE, "csrc", "libspk_b200.so")   # override: A/B builds

SPK_OK = 0
ACT_NONE, ACT_SILU, ACT_SSP, ACT_GIVEN = 0, 1, 2, 3
SAVE_DERIV = 0x10
RBF_GAUSSIAN, RBF_BESSEL = 0, 1
GEO_STRIDE = 8

P = c_void_p  # device pointers and the stream travel as void*

class NHCParams(Structure):
    """spk_nhc_params_t of include/spk_b200.h."""
    _fields_ = [("chain_length", c_int32), ("multi_step", c_int32), ("order", c_int32), ("massive", c_int32),
                ("kb_temperature", c_double), ("time_step", c_double * 7)]


class NHCBarostat(Structure):
    """spk_nhc_barostat_t of include/spk_b200.h (parameters and device pointers of the chain / cell state)."""
    _fields_ = [("anisotropic", c_int32), ("massive", c_int32), ("chain_length", c_int32), ("multi_step", c_int32),
                ("order", c_int32), ("reserved", c_int32), ("kb_temperature", c_double), ("time_step", c_double),
                ("target_pressure", c_double), ("ys_time_step", c_double * 7),
                ("t_v", c_void_p), ("t_f", c_void_p), ("t_m", c_void_p), ("c_v", c_void_p), ("c_f", c_void_p),
                ("c_m", c_void_p), ("b_v", c_void_p), ("b_f", c_void_p), ("b_m", c_void_p)]


class HeadTail(Structure):
    """spk_head_tail_t of include/spk_b200.h."""
    _fields_ = [("wmix", c_void_p), ("w0", c_void_p), ("w0t", c_void_p), ("b0", c_void_p), ("w1", c_void_p),
                ("b1", c_void_p), ("Fi", c_int32), ("H", c_int32), ("act", c_int32), ("reserved", c_int32)]


class LBFGSState(Structure):
    """spk_lbfgs_t of include/spk_b200.h (device pointers of the optimizer state and its parameters)."""
    _fields_ = [("r", c_void_p), ("r0", c_void_p), ("f0", c_void_p), ("s", c_void_p), ("y", c_void_p),
                ("rho", c_void_p), ("p", c_void_p), ("counter", c_void_p), ("fmax", c_void_p), ("fmax_sys", c_void_p),
                ("converged", c_void_p), ("steps", c_void_p), ("n_unconverged", c_void_p), ("fixed", c_void_p),
                ("model_positions", c_void_p), ("sys_ptr", c_void_p), ("order", c_void_p), ("n_atoms", c_int64),
                ("n_sys", c_int64), ("n_warp", c_int64), ("memory", c_int64), ("force_conversion", c_double),
                ("position_conversion", c_double), ("maxstep", c_double), ("damping", c_double), ("h0", c_double)]


class PairParams(Structure):
    """spk_pair_t of include/spk_b200.h."""
    _fields_ = [("kind", c_int32), ("n_terms", c_int32), ("a_pow", c_void_p), ("a_div", c_void_p),
                ("coefficients", c_void_p), ("exponents", c_void_p), ("ke", c_double), ("cutoff", c_double),
                ("shift", c_double), ("switch_on", c_double), ("switch_off", c_double), ("d_max", c_double),
                ("alpha", c_double)]


PAIR_ZBL, PAIR_COULOMB, PAIR_DAMPED_COULOMB, PAIR_EWALD_REAL = 0, 1, 2, 3     # SPK_PAIR_*
PAIR_MAX_TERMS = 16                                       # SPK_PAIR_MAX_TERMS

class VibParams(Structure):
    """spk_vib_t of include/spk_b200.h (device pointers of the replica batch and the vibrational-analysis buffers)."""
    _fields_ = [("base", c_void_p), ("positions", c_void_p), ("steps", c_void_p), ("counter", c_void_p),
                ("forces", c_void_p), ("dipole", c_void_p), ("polar", c_void_p), ("idx_m", c_void_p),
                ("sys_ptr", c_void_p), ("n_displaced", c_void_p), ("hess_ptr", c_void_p), ("masses", c_void_p),
                ("h_raw", c_void_p),
                ("hessian", c_void_p), ("hessian_mw", c_void_p), ("dipole_deriv", c_void_p), ("polar_deriv", c_void_p),
                ("n_atoms", c_int64), ("n_sys", c_int64), ("n_cols", c_int64), ("nfree", c_int64),
                ("max_atoms", c_int64), ("delta", c_double), ("mw_scale", c_double)]


class PhononParams(Structure):
    """spk_ph_t of include/spk_b200.h (the supercell layout, force-constant and minimum-image buffers of a phonon run)."""
    _fields_ = [("h_raw", c_void_p), ("force_constants", c_void_p), ("work", c_void_p), ("prim_ptr", c_void_p),
                ("fc_ptr", c_void_p), ("lattice", c_void_p), ("neg", c_void_p), ("positions", c_void_p),
                ("cell", c_void_p), ("super_cell", c_void_p), ("super_inv", c_void_p), ("heights", c_void_p),
                ("masses", c_void_p), ("img_count", c_void_p), ("img_lattice", c_void_p), ("supercell", c_int32 * 9),
                ("n_sys", c_int64), ("n_prim", c_int64), ("n_rows", c_int64), ("n_cells", c_int64),
                ("max_atoms", c_int64), ("rounds", c_int64), ("acoustic", c_int32), ("reserved", c_int32),
                ("tie_tol", c_double), ("mw_scale", c_double)]


PH_MAX_IMAGES = 8           # SPK_PH_MAX_IMAGES
PH_THERMO_FIELDS = 6        # spk_ph_thermo: zero-point energy, F, S, C_v, modes left out, imaginary modes


class FIREState(Structure):
    """spk_fire_t of include/spk_b200.h (device pointers of the FIRE state, the filter settings and the parameters)."""
    _fields_ = [("s", c_void_p), ("r", c_void_p), ("v", c_void_p), ("g", c_void_p), ("h", c_void_p), ("hv", c_void_p),
                ("hg", c_void_p), ("cell0", c_void_p), ("cell_factor", c_void_p), ("dt", c_void_p), ("a", c_void_p),
                ("nsteps", c_void_p), ("started", c_void_p), ("sums", c_void_p), ("coef", c_void_p),
                ("workspace", c_void_p), ("counter", c_void_p), ("fmax", c_void_p), ("fmax_sys", c_void_p),
                ("converged", c_void_p), ("steps", c_void_p), ("n_unconverged", c_void_p), ("fixed", c_void_p),
                ("model_positions", c_void_p), ("model_cell", c_void_p), ("idx_m", c_void_p), ("sys_ptr", c_void_p),
                ("mask", c_double * 9), ("n_atoms", c_int64), ("n_sys", c_int64), ("nmin", c_int64),
                ("filter", c_int32), ("hydrostatic_strain", c_int32), ("constant_volume", c_int32),
                ("reserved", c_int32), ("force_conversion", c_double), ("energy_conversion", c_double),
                ("position_conversion", c_double), ("scalar_pressure", c_double), ("maxstep", c_double),
                ("dtmax", c_double), ("finc", c_double), ("fdec", c_double), ("astart", c_double), ("fa", c_double)]


class NEBState(Structure):
    """spk_neb_t of include/spk_b200.h (device pointers of the band layout and the NEB buffers, and the parameters)."""
    _fields_ = [("r", c_void_p), ("r_initial", c_void_p), ("r_final", c_void_p), ("end_energies", c_void_p),
                ("climb", c_void_p), ("fixed", c_void_p), ("idx_img", c_void_p), ("img_ptr", c_void_p),
                ("band_ptr", c_void_p), ("coef", c_void_p), ("diag", c_void_p), ("climbing", c_void_p),
                ("neb_forces", c_void_p), ("workspace", c_void_p), ("n_atoms", c_int64), ("n_images", c_int64),
                ("n_bands", c_int64), ("k", c_double), ("force_conversion", c_double),
                ("energy_conversion", c_double)]


FIRE_COEF = 7               # step coefficients per system (spk_fire_t.coef)
NEB_COEF, NEB_DIAG = 3, 6   # per interior image: spk_neb_t.coef and spk_neb_t.diag
RELAX_WARP_ATOMS = 256      # SPK_RELAX_WARP_ATOMS
RELAX_MAX_MEMORY = 4096     # SPK_RELAX_MAX_MEMORY


# name -> argument ctypes (return type is int unless listed in _RESTYPE)
SIGNATURES = {
    "spk_version": [],
    "spk_graph_workspace_bytes": [c_int64, c_int64],
    "spk_graph_build": [P, P, c_int64, c_int64, P, P, P, P, P, P, P, P, c_size_t, P],
    "spk_graph_build_active": [P, P, P, c_float, c_int64, c_int64, P, P, P, P, P, P, P, P, c_size_t, P],
    "spk_segment_ptr": [P, c_int64, c_int64, P, P],
    "spk_pairwise_fwd": [P, P, P, P, c_int64, c_int64, P, P],
    "spk_pairwise_bwd": [P, P, P, P, P, c_int64, c_float, P, P],
    "spk_edge_geometry": [P, P, c_int64, c_int, c_int, P, P, c_float, P, P, P, P, P],
    "spk_rbf_fwd": [P, c_int64, c_int, c_int, P, P, P, P, P],
    "spk_cosine_cutoff_fwd": [P, c_int64, c_float, P, P, P],
    "spk_act_fwd": [P, c_int64, c_int, P, P, P],
    "spk_embedding": [P, P, c_int64, c_int, c_int, P, P],
    "spk_segment_sum": [P, P, P, c_int64, c_int, P, P],
    "spk_dense": [P, c_int64, c_int, c_int64, P, c_int, P, c_int, P, c_int, P, c_int64, P, c_int64, P, P],
    "spk_tc_packed_floats": [c_int, c_int],
    "spk_tc_pack_weight": [P, c_int, c_int, P, P],
    "spk_dense_tc": [P, c_int64, c_int, c_int64, P, c_int, P, c_int, P, c_int, P, c_int64, P, c_int64, P, P],
    "spk_painn_edge_fwd": [P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, P, P, P],
    "spk_painn_edge_bwd": [P, P, P, P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, P, P, P, c_int, P],
    "spk_painn_filter_packed_floats": [],
    "spk_painn_pack_filter": [P, P, c_int, c_int, P, P],
    "spk_painn_edge_fwd_tc": [P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, P, P, P],
    "spk_painn_edge_bwd_tc": [P, P, P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, P, P, P, c_int, P],
    "spk_painn_edge_wij_fwd": [P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, P, P, P],
    "spk_painn_edge_wij_bwd": [P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, P, P, P, P, P],
    "spk_painn_mix_ctx": [P, P, c_int64, c_int, c_float, P, P],
    "spk_painn_mix_update": [P, P, P, P, c_int64, c_int, P, P, P],
    "spk_painn_mix_update_bwd": [P, P, P, P, c_int64, c_int, P, P, P],
    "spk_painn_mix_ctx_bwd": [P, P, P, c_int64, c_int, c_float, P, P, P],
    "spk_cfconv_fwd": [P, P, P, P, P, c_int64, c_int64, c_int, P, P],
    "spk_schnet_filter_packed_floats": [],
    "spk_schnet_pack_filter": [P, P, P, c_int, c_int, P, P],
    "spk_schnet_cfconv_fwd_tc": [P, P, P, P, P, P, P, c_int, c_int64, c_int64, c_int, c_int, P, P],
    "spk_cfconv_bwd": [P, P, P, P, P, P, P, c_int64, c_int64, c_int, P, P, P, P],
    "spk_radial_bwd": [P, P, P, P, P, c_int64, c_int, P, c_int, P],
    "spk_atomwise_out": [P, P, P, P, c_int64, c_int64, c_int, P, P, P],
    "spk_atomwise_out_bwd": [P, P, P, c_int64, c_int, P, P],
    "spk_add": [P, P, c_int64, P, P],
    "spk_halo_pull": [P, P, P, P, c_int64, c_int, P],
    "spk_halo_pull_add": [P, P, P, P, P, P, c_int64, c_int, P],
    "spk_md_velocity_verlet": [P, P, P, P, P, c_int64, c_float, c_float, c_float, c_int, P],
    "spk_neighbor_list_workspace_bytes": [c_int64, c_int64],
    "spk_neighbor_list": [P, P, P, P, c_int64, c_int64, c_float, c_int64, c_int, P, P, P, P, P, P, c_size_t, P],
    "spk_md_thermostat_workspace_bytes": [c_int64, c_int64],
    "spk_md_kinetic_energy": [P, P, P, P, c_int64, c_int64, c_double, P, P, P, c_size_t, P],
    "spk_md_berendsen": [P, P, P, P, c_int64, c_int64, c_double, c_double, c_double, P, c_size_t, P],
    "spk_md_nhc": [P, P, P, P, c_int64, c_int64, POINTER(NHCParams), P, P, P, P, c_size_t, P],
    "spk_md_langevin": [P, P, c_int64, c_double, c_double, c_double, c_uint64, P, P],
    "spk_philox4x32_10": [c_uint64, P, c_int64, P, P],
    "spk_pairwise_virial_workspace_bytes": [c_int64, c_int64],
    "spk_pairwise_virial": [P, P, P, P, P, c_int64, c_int64, P, P, c_size_t, P],
    "spk_md_barostat_workspace_bytes": [c_int64, c_int64],
    "spk_md_kinetic_energy_tensor": [P, P, P, P, c_int64, c_int64, P, P, c_size_t, P],
    "spk_md_barostat_thermostat": [POINTER(NHCBarostat), P, P, P, P, c_int64, c_int64, P, c_size_t, P],
    "spk_md_barostat_kick": [POINTER(NHCBarostat), P, P, P, P, c_int64, c_int64, P, P, c_double, P, c_size_t, P],
    "spk_md_barostat_half_step": [POINTER(NHCBarostat), P, P, c_double, P, P, c_int64, c_int64, P, c_size_t, P],
    "spk_md_barostat_main_step": [POINTER(NHCBarostat), P, P, P, P, P, P, c_int64, c_int64, P, P, c_double, P, c_size_t,
                                  P],
    "spk_rpmd_workspace_bytes": [c_int64, c_int64],
    "spk_rpmd_normal_modes": [P, P, c_int64, c_int32, P, c_int32, P],
    "spk_rpmd_main_step": [P, P, P, P, c_int64, c_int32, P, P, c_double, P],
    "spk_rpmd_pile": [P, P, P, P, c_int64, c_int64, c_int32, P, P, P, c_double, c_int32, c_uint64, P, P, c_size_t, P],
    "spk_rpmd_nhc": [P, P, P, P, c_int64, c_int64, c_int32, P, POINTER(NHCParams), c_int32, P, P, P, P, c_size_t, P],
    "spk_rpmd_gle": [P, P, c_int64, c_int32, P, P, P, c_int32, c_int32, P, c_uint64, P, c_int32, P],
    "spk_rpmd_barostat_workspace_bytes": [c_int64, c_int64],
    "spk_so3_conv_fwd": [P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, c_int, P, P],
    "spk_so3_conv_bwd": [P, P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, c_int, P, P, P, c_int, P],
    "spk_so3_tp_fwd": [P, P, c_int64, c_int, c_int, P, P],
    "spk_so3_tp_bwd": [P, P, P, c_int64, c_int, c_int, P, P, P],
    "spk_so3_gate_fwd": [P, P, c_int64, c_int, c_int, P, P],
    "spk_so3_gate_bwd": [P, P, P, c_int64, c_int, c_int, P, P, P, P],
    "spk_so3_put_l0": [P, P, c_int64, c_int, c_int, P, P],
    "spk_so3_take_l0": [P, c_int64, c_int, c_int, P, P],
    "spk_md_property": [P, c_int64, c_float, P, P],
    "spk_md_record": [P, c_int64, P, c_int64, c_int64, P, P],
    "spk_md_record_advance": [P, c_int64, c_int64, P],
    "spk_geq_ctx": [P, P, c_int64, c_int, c_int, P, P],
    "spk_geq_ctx_bwd": [P, P, c_int64, c_int, c_int, P, P, P],
    "spk_geq_gate": [P, P, c_int64, c_int, c_int, P, P, P],
    "spk_geq_gate_bwd": [P, P, P, P, c_int64, c_int, c_int, P, P, P],
    "spk_head_workspace_bytes": [c_int64, c_int64],
    "spk_head_fwd": [c_int, POINTER(HeadTail), P, P, P, P, P, P, P, c_int64, c_int64, c_int, c_int, P, P, P, P, c_size_t,
                     P],
    "spk_head_charges": [P, P, P, c_int64, P, P],
    "spk_head_bwd": [c_int, POINTER(HeadTail), P, P, P, P, P, P, c_int64, c_int, c_int, P, P, P, P],
    "spk_head_scalar_bwd": [P, P, P, P, P, c_int, c_int, P, c_int64, c_int, P, P, P],
    "spk_rpmd_barostat_thermostat": [P, c_int64, c_double, P, c_uint64, P, P],
    "spk_rpmd_barostat_half_step": [P, P, c_double, P, P, P, c_int64, c_int64, c_int32, P, P, P, c_double, c_double,
                                    c_double, c_double, P, P, P, c_size_t, P],
    "spk_rpmd_barostat_main_step": [P, P, P, P, P, c_int64, c_int64, c_int32, P, P, c_double, P, P, P, P, c_double, P,
                                    c_size_t, P],
    "spk_head_charges_bwd_workspace_bytes": [c_int64, c_int64],
    "spk_head_charges_bwd": [P, P, P, c_int64, c_int64, c_int, P, P, c_size_t, P],
    "spk_head_bwd_q": [c_int, POINTER(HeadTail), P, P, P, P, P, P, P, c_int64, c_int, c_int, P, P, P, P],
    "spk_head_scalar_bwd_q": [P, P, P, P, P, P, c_int, c_int, P, c_int64, c_int, P, P, P],
    "spk_pair_energy_workspace_bytes": [c_int64, c_int64],
    "spk_pair_energy_fwd": [POINTER(PairParams), P, P, P, P, P, P, P, P, P, c_int64, c_int64, P, P, c_size_t, P],
    "spk_pair_energy_bwd": [POINTER(PairParams), P, P, P, P, P, P, P, P, P, P, P, P, P, c_int64, c_int64, P, P, P],
    "spk_ewald_workspace_bytes": [c_int64, c_int64, c_int64],
    "spk_ewald_fwd": [P, P, P, P, P, P, c_int64, c_int64, c_int64, c_double, c_double, P, P, P, c_size_t, P],
    "spk_ewald_bwd": [P, P, P, P, P, P, c_int64, c_int64, c_int64, c_double, c_double, P, P, P, c_int, P, P, c_int, P,
                      c_size_t, P],
    "spk_pairwise_virial_add": [P, P, P, P, P, c_int64, c_int64, P, P, c_size_t, P],
    "spk_relax_step": [POINTER(LBFGSState), P, P],
    "spk_relax_converged": [POINTER(LBFGSState), P, P],
    "spk_ensemble_workspace_bytes": [c_int64, c_int64],
    "spk_ensemble_moments": [P, c_int64, c_int64, c_int, c_double, c_double, P, P, P, P],
    "spk_ensemble_forces": [P, c_int64, P, P, c_int64, c_int64, c_double, c_double, P, P, P, P, c_size_t, P],
    "spk_ensemble_uncertainty": [P, c_double, P, P, P, c_double, c_int64, c_int64, c_int, c_double, c_double, c_double, P,
                                 P, P],
    "spk_vib_displace": [POINTER(VibParams), P],
    "spk_vib_assemble": [POINTER(VibParams), P],
    "spk_vib_finish": [POINTER(VibParams), P],
    "spk_ph_force_constants": [POINTER(PhononParams), P],
    "spk_ph_images": [POINTER(PhononParams), P],
    "spk_ph_dynmat": [POINTER(PhononParams), P, c_int64, P, P, P],
    "spk_ph_dos": [P, c_int64, c_int64, P, c_int64, P, c_int64, c_double, P, P],
    "spk_ph_thermo_workspace_bytes": [c_int64, c_int64],
    "spk_ph_thermo": [P, c_int64, c_int64, P, c_int64, P, c_int64, P, c_int64, c_double, c_double, c_double, P, P,
                      c_size_t, P],
    "spk_md_record_velocities": [P, P, c_int64, P, c_int64, c_int64, P, P],
    "spk_spectrum_workspace_bytes": [c_int64, c_int64, c_int64],
    "spk_spectrum_series": [P, c_int64, c_int64, c_int64, P, P, c_int64, c_int, c_double, P, P, P, P],
    "spk_spectrum_autocorrelation": [P, c_int64, P, P, c_int64, c_int64, P, P, c_size_t, P],
    "spk_spectrum_transform": [P, c_int64, c_int64, P, c_double, P, P, c_size_t, P],
    "spk_spectrum_stream_state_bytes": [c_int64, c_int64],
    "spk_spectrum_stream_finalise_workspace_bytes": [c_int64, c_int64],
    "spk_spectrum_stream_push": [P, P, c_int64, c_int64, P, P, c_int64, c_int, c_double, P, c_int64, c_int64, P, P],
    "spk_spectrum_stream_finalise": [P, c_int64, c_int64, c_int64, P, c_int64, P, P, c_int64, c_int64, P, P, c_size_t,
                                     P],
    "spk_fire_workspace_bytes": [c_int64, c_int64],
    "spk_fire_forces": [POINTER(FIREState), P, P, P],
    "spk_fire_step": [POINTER(FIREState), P],
    "spk_neb_workspace_bytes": [c_int64, c_int64],
    "spk_neb_forces": [POINTER(NEBState), P, P, P],
    "spk_md_motion_workspace_bytes": [c_int64, c_int64],
    "spk_md_remove_motion": [P, P, P, P, P, P, c_int64, c_int64, c_int, c_float, P, c_int64, P, c_size_t, P],
    "spk_md_wrap_positions": [P, P, P, c_int64, c_int32, P, c_int64, P, c_int64, c_double, c_float, P, c_int64, P],
    "spk_md_initial_momenta": [P, P, P, P, c_int64, c_int64, c_int, c_double, P, c_uint64, P, c_size_t, P],
    "spk_md_step_advance": [P, P],
    "spk_pme_workspace_bytes": [c_int64, c_int64, c_int64, c_int64, c_int64, c_int],
    "spk_pme_spread": [P, P, P, P, P, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, P, P, c_size_t, P],
    "spk_pme_energy": [P, P, P, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_double, c_double, P, P, P, P,
                       c_size_t, P],
    "spk_pme_bwd": [P, P, P, P, P, c_int64, c_int64, c_int64, c_int64, c_int64, c_int, c_double, c_double, P, P, P, c_int,
                    P, P, c_int, P, c_size_t, P],
}
_RESTYPE = {"spk_graph_workspace_bytes": c_size_t, "spk_tc_packed_floats": c_size_t,
            "spk_pairwise_virial_workspace_bytes": c_size_t, "spk_md_barostat_workspace_bytes": c_size_t,
            "spk_schnet_filter_packed_floats": c_size_t,
            "spk_painn_filter_packed_floats": c_size_t, "spk_neighbor_list_workspace_bytes": c_size_t,
            "spk_md_thermostat_workspace_bytes": c_size_t, "spk_rpmd_workspace_bytes": c_size_t,
            "spk_rpmd_barostat_workspace_bytes": c_size_t, "spk_head_workspace_bytes": c_size_t,
            "spk_head_charges_bwd_workspace_bytes": c_size_t, "spk_pair_energy_workspace_bytes": c_size_t,
            "spk_ewald_workspace_bytes": c_size_t, "spk_ensemble_workspace_bytes": c_size_t,
            "spk_spectrum_workspace_bytes": c_size_t, "spk_fire_workspace_bytes": c_size_t,
            "spk_md_motion_workspace_bytes": c_size_t, "spk_spectrum_stream_state_bytes": c_size_t,
            "spk_spectrum_stream_finalise_workspace_bytes": c_size_t, "spk_neb_workspace_bytes": c_size_t,
            "spk_pme_workspace_bytes": c_size_t, "spk_ph_thermo_workspace_bytes": c_size_t}

_lib = None


class SpkLibraryError(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle; raises SpkLibraryError if the CUDA library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SpkLibraryError(
            f"{LIB_PATH} not found: build it with `python -m schnetpack_b200.build` (needs nvcc). "
            "schnetpack_b200 has no CPU fallback."
        )
    h = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(h, name)  # AttributeError if the .so is stale / symbol missing
        fn.argtypes = argtypes
        fn.restype = _RESTYPE.get(name, c_int)
    _lib = h
    return h


def check(rc: int, name: str):
    if rc == SPK_OK:
        return
    if rc == -1:
        raise ValueError(f"{name}: invalid argument (SPK_ERR_ARG)")
    if rc == -2:
        raise NotImplementedError(f"{name}: shape outside the compiled sm_90a templates (SPK_ERR_UNSUPPORTED)")
    raise RuntimeError(f"{name}: CUDA error {-rc - 1000}")


# kernels launched per C-ABI call (default 1); bench.py reports the running total as ``gpu_launches``
LAUNCHES = {"spk_graph_build": 8, "spk_graph_build_active": 8, "spk_atomwise_out": 2, "spk_neighbor_list": 6,
            "spk_md_kinetic_energy": 2, "spk_md_berendsen": 3, "spk_pairwise_virial": 2,
            "spk_md_kinetic_energy_tensor": 3, "spk_md_barostat_thermostat": 4, "spk_md_barostat_kick": 3,
            "spk_md_barostat_half_step": 2, "spk_md_barostat_main_step": 2, "spk_rpmd_barostat_half_step": 2,
            "spk_rpmd_barostat_main_step": 2, "spk_head_fwd": 2,
            "spk_relax_converged": 2, "spk_pair_energy_fwd": 2, "spk_head_charges_bwd": 3,
            "spk_pairwise_virial_add": 2, "spk_spectrum_autocorrelation": 2, "spk_spectrum_transform": 2,
            "spk_fire_forces": 3, "spk_fire_step": 2, "spk_md_remove_motion": 3, "spk_spectrum_stream_push": 2,
            "spk_spectrum_stream_finalise": 2, "spk_neb_forces": 3, "spk_pme_spread": 8,
            "spk_pme_energy": 2, "spk_pme_bwd": 2, "spk_ph_thermo": 2}
# spk_pme_spread: 4 without atoms (cell, setup, scan, spread); spk_pme_bwd: 1 per part present (atoms, cell or virial);
# spk_ph_force_constants: 1 + the rounds run;
# spk_relax_step: 1 per size path present; spk_rpmd_pile / spk_rpmd_nhc: 3 if global; spk_md_initial_momenta: 4 if uniform
MOTION_CENTER_OF_MASS, MOTION_TRANSLATION, MOTION_ROTATION = 1, 2, 4       # SPK_MOTION_*
launch_count = 0


def call(name: str, *args, launches: Optional[int] = None):
    """``launches``: kernels this call enqueues when it differs from the entry point's usual count in LAUNCHES"""
    global launch_count
    rc = getattr(lib(), name)(*args)
    check(rc, name)
    launch_count += LAUNCHES.get(name, 1) if launches is None else launches

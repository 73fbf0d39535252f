"""Keys of the tensor dictionary exchanged between modules -- the reference's boundary contract, reused verbatim
(/root/reference/src/schnetpack/properties.py:10-40) so that batches built for the reference feed these modules."""
idx = "_idx"
Z = "_atomic_numbers"
position = "_positions"
R = position
cell = "_cell"
strain = "strain"
pbc = "_pbc"
seg_m = "_seg_m"
idx_m = "_idx_m"
idx_i = "_idx_i"
idx_j = "_idx_j"
idx_i_lr = "_idx_i_lr"
idx_j_lr = "_idx_j_lr"
lidx_i = "_idx_i_local"
lidx_j = "_idx_j_local"
Rij = "_Rij"
Rij_lr = "_Rij_lr"
n_atoms = "_n_atoms"
offsets = "_offsets"
offsets_lr = "_offsets_lr"
R_strained = position + "_strained"
cell_strained = cell + "_strained"
n_nbh = "_n_nbh"
energy = "energy"
forces = "forces"
stress = "stress"
masses = "masses"
total_charge = "total_charge"
dipole_moment = "dipole_moment"
partial_charges = "partial_charges"
polarizability = "polarizability"
# opt-in input of this package (not a reference key): a caller-owned fp64 [n_sys, 3, 3] buffer under this key makes the
# backward of PairwiseDistances write the per-system virial W = sum_e dE/dr_e (x) r_e into it (stress = W / V)
virial = "_virial"
# set by FilterShortRange (not a reference key): the short-range keys keep the full list, and pair terms that read it
# mask d > short_range_cutoff (a CPU scalar tensor, so reading it is no device sync)
short_range_cutoff = "_short_range_cutoff"
# set by PairwiseDistances when a virial is requested (not a reference key): the state its backward shares with terms
# that deposit a virial of their own first (the reciprocal Ewald term)
virial_sink = "_virial_sink"

"""ctypes binding of the C-ABI library ``csrc/libspk_b200.so``, read from its header ``include/spk_b200.h``.

The header is the only statement of the ABI.  At import, ``read_header`` turns its parameter structs into ctypes
Structures (STRUCTS), its prototypes into argument and return types (SIGNATURES, RESTYPE) and its integer ``SPK_*``
defines into CONSTANTS; a construct outside that small grammar raises, naming the declaration, instead of being bound
wrong.  To add an entry point, declare it in the header; this module needs an edit only when the entry point launches
more than one kernel (LAUNCHES).

There is NO fallback: if the library is missing (not built) importing any op raises, and every op raises when it is
handed a non-CUDA tensor.  torch is used only as the owner of device memory and streams.
"""
from __future__ import annotations

import ctypes
import os
import re
from ctypes import POINTER, Structure, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_uint64, c_void_p
from typing import Optional

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("SPK_B200_LIB") or os.path.join(HERE, "csrc", "libspk_b200.so")   # override: A/B builds
HEADER = os.path.join(HERE, "..", "include", "spk_b200.h")

P = c_void_p  # device pointers and the stream travel as void*

_SCALARS = {"int": c_int, "int32_t": c_int32, "int64_t": c_int64, "uint64_t": c_uint64, "size_t": c_size_t,
            "float": c_float, "double": c_double}
_POINTEES = {"void", "uint8_t", "uint32_t", *_SCALARS}     # element types a void* argument or field may point to
_RESTYPES = {"int": c_int, "size_t": c_size_t}
_STRUCT = re.compile(r"typedef\s+struct\s*\{([^{}]*)\}\s*(\w+)\s*;")


def read_header(text: str):
    """(STRUCTS, SIGNATURES, RESTYPE, CONSTANTS) of the C ABI declared in ``text``; raises ValueError, naming the
    declaration, on a type or declaration outside the header's grammar."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    constants = {}
    for name, value in re.findall(r"^[ \t]*#[ \t]*define[ \t]+(SPK_\w+)[ \t]+(.*?)[ \t]*$", text, flags=re.M):
        literal = re.fullmatch(r"\(?(-?(?:0[xX][0-9a-fA-F]+|\d+))[uUlL]*\)?", value)   # function-like macros never match
        if literal:
            constants[name] = int(literal.group(1), 0)
    text = re.sub(r"^[ \t]*#.*$", "", text, flags=re.M)

    structs = {}

    def ctype(base, star, decl):
        if star and base in structs:
            return POINTER(structs[base])
        if star and base in _POINTEES:
            return c_void_p
        if not star and base in _SCALARS:
            return _SCALARS[base]
        if not star and base == "spk_stream_t":
            return c_void_p
        raise ValueError(f"spk_b200.h: unknown type '{base}{star}' in '{decl}'")

    for body, name in _STRUCT.findall(text):
        fields = []
        for decl in filter(None, (" ".join(d.split()) for d in body.split(";"))):
            base, declarators = re.fullmatch(r"(?:const )?(\w*) ?(.*)", decl).groups()
            for part in declarators.split(","):
                field = re.fullmatch(r"(\*?) ?(\w+) ?(?:\[(\d+)\])?", part.strip())
                if not field:
                    raise ValueError(f"spk_b200.h: cannot read the field declaration '{decl}' of {name}")
                t = ctype(base, field.group(1), decl)
                fields.append((field.group(2), t * int(field.group(3)) if field.group(3) else t))
        structs[name] = type(name, (Structure,), {"_fields_": fields})

    signatures, restype = {}, {}
    for decl in (" ".join(d.split()) for d in _STRUCT.sub("", text).split(";")):
        if "(" not in decl:
            continue
        proto = re.fullmatch(r"(\w+) (spk_\w+) ?\((.*)\)", decl)
        if not proto:
            raise ValueError(f"spk_b200.h: cannot read the declaration '{decl}'")
        ret, name, params = proto.groups()
        if ret not in _RESTYPES:
            raise ValueError(f"spk_b200.h: {name} returns '{ret}', not int or size_t")
        argtypes = []
        for param in ([] if params.strip() == "void" else params.split(",")):
            arg = re.fullmatch(r"(?:const )?(\w+)( ?\* ?| )\w+", param.strip())
            if not arg:
                raise ValueError(f"spk_b200.h: cannot read the parameter '{param.strip()}' of {name}")
            argtypes.append(ctype(arg.group(1), arg.group(2).strip(), decl))
        signatures[name], restype[name] = argtypes, _RESTYPES[ret]
    return structs, signatures, restype, constants


with open(HEADER) as _f:
    STRUCTS, SIGNATURES, RESTYPE, CONSTANTS = read_header(_f.read())


def _defines(*names):
    return [CONSTANTS["SPK_" + name] for name in names]


NHCParams = STRUCTS["spk_nhc_params_t"]
NHCBarostat = STRUCTS["spk_nhc_barostat_t"]
HeadTail = STRUCTS["spk_head_tail_t"]
LBFGSState = STRUCTS["spk_lbfgs_t"]
PairParams = STRUCTS["spk_pair_t"]
VibParams = STRUCTS["spk_vib_t"]
PhononParams = STRUCTS["spk_ph_t"]
FIREState = STRUCTS["spk_fire_t"]
NEBState = STRUCTS["spk_neb_t"]

SPK_OK, SPK_ERR_ARG, SPK_ERR_UNSUPPORTED = _defines("OK", "ERR_ARG", "ERR_UNSUPPORTED")
ACT_NONE, ACT_SILU, ACT_SSP, ACT_GIVEN = _defines("ACT_NONE", "ACT_SILU", "ACT_SSP", "ACT_GIVEN")
SAVE_DERIV, GEO_STRIDE = _defines("SAVE_DERIV", "GEO_STRIDE")
RBF_GAUSSIAN, RBF_BESSEL = _defines("RBF_GAUSSIAN", "RBF_BESSEL")
PAIR_ZBL, PAIR_COULOMB, PAIR_DAMPED_COULOMB, PAIR_EWALD_REAL, PAIR_MAX_TERMS = _defines(
    "PAIR_ZBL", "PAIR_COULOMB", "PAIR_DAMPED_COULOMB", "PAIR_EWALD_REAL", "PAIR_MAX_TERMS")
PH_MAX_IMAGES, RELAX_WARP_ATOMS, RELAX_MAX_MEMORY = _defines("PH_MAX_IMAGES", "RELAX_WARP_ATOMS", "RELAX_MAX_MEMORY")
MOTION_CENTER_OF_MASS, MOTION_TRANSLATION, MOTION_ROTATION = _defines(
    "MOTION_CENTER_OF_MASS", "MOTION_TRANSLATION", "MOTION_ROTATION")

PH_THERMO_FIELDS = 6        # spk_ph_thermo: zero-point energy, F, S, C_v, modes left out, imaginary modes
FIRE_COEF = 7               # step coefficients per system (spk_fire_t.coef)
NEB_COEF, NEB_DIAG = 3, 6   # per interior image: spk_neb_t.coef and spk_neb_t.diag

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
        fn.restype = RESTYPE[name]
    _lib = h
    return h


def check(rc: int, name: str):
    if rc == SPK_OK:
        return
    if rc == SPK_ERR_ARG:
        raise ValueError(f"{name}: invalid argument (SPK_ERR_ARG)")
    if rc == SPK_ERR_UNSUPPORTED:
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
            "spk_pme_energy": 2, "spk_pme_bwd": 2, "spk_ph_thermo": 2, "spk_rdf_accumulate": 7,
            "spk_msd_accumulate": 7, "spk_md_nhc_per_system": 3, "spk_remd_exchange": 2}
# spk_pme_spread: 4 without atoms (cell, setup, scan, spread); spk_pme_bwd: 1 per part present (atoms, cell or virial);
# spk_ph_force_constants: 1 + the rounds run;
# spk_rdf_accumulate: 2 without atoms (gate, fold); spk_msd_accumulate: 5 without remove_com;
# spk_relax_step: 1 per size path present; spk_rpmd_pile / spk_rpmd_nhc: 3 if global; spk_md_initial_momenta: 4 if uniform
# spk_md_nhc_per_system: 1 if massive (no kinetic-energy passes)
launch_count = 0


def call(name: str, *args, launches: Optional[int] = None):
    """``launches``: kernels this call enqueues when it differs from the entry point's usual count in LAUNCHES"""
    global launch_count
    rc = getattr(lib(), name)(*args)
    check(rc, name)
    launch_count += LAUNCHES.get(name, 1) if launches is None else launches

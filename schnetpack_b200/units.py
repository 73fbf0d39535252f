"""Unit conversion of the reference (units.py:132-189) without ``ase``: ``convert_units(src, tgt)`` parses unit strings
such as ``"kcal / mol"`` or ``"Bohr"`` into ASE's frame (eV, Angstrom, amu) and returns the factor src / tgt.

The unit names and values are those of ASE's units module for CODATA 2014 (the constants ``md.py`` builds its MD units
from), so that a conversion here gives the number the reference computes."""
from __future__ import annotations

import math
import re
from typing import Union

__all__ = ["convert_units"]

# CODATA 2014 (ase/units.py, CODATA['2014'])
_c = 299792458.0
_mu0 = 4e-7 * math.pi
_hplanck = 6.626070040e-34
_e = 1.6021766208e-19
_me = 9.10938356e-31
_mp = 1.672621898e-27
_Nav = 6.022140857e23
_k = 1.38064852e-23
_amu = 1.660539040e-27
_eps0 = 1.0 / _mu0 / _c ** 2
_hbar = _hplanck / (2.0 * math.pi)


def _ase_units() -> dict:
    """The unit table of ase.units.create_units('2014')."""
    u = dict(_c=_c, _mu0=_mu0, _hplanck=_hplanck, _e=_e, _me=_me, _mp=_mp, _Nav=_Nav, _k=_k, _amu=_amu, _eps0=_eps0,
             _hbar=_hbar)
    u["Ang"] = u["Angstrom"] = 1.0
    u["nm"] = 10.0
    u["um"] = 1e4
    u["mm"] = 1e7
    u["cm"] = 1e8
    u["m"] = 1e10
    u["eV"] = 1.0
    u["second"] = 1e10 * math.sqrt(_e / _amu)
    u["fs"] = 1e-15 * u["second"]
    u["kB"] = _k / _e
    u["Pascal"] = (1.0 / _e) / 1e30
    u["GPa"] = 1e9 * u["Pascal"]
    u["bar"] = 1e5 * u["Pascal"]
    u["Debye"] = 1.0 / 1e11 / _e / _c
    u["alpha"] = _e ** 2 / (4 * math.pi * _eps0) / _hbar / _c
    u["invcm"] = 100 * _c * _hplanck / _e
    u["_aut"] = _hbar / (u["alpha"] ** 2 * _me * _c ** 2)
    u["_auv"] = _e ** 2 / _hbar / (4 * math.pi * _eps0)
    u["_auf"] = u["alpha"] ** 3 * _me ** 2 * _c ** 3 / _hbar
    u["_aup"] = u["alpha"] ** 5 * _me ** 4 * _c ** 5 / _hbar ** 3
    u["AUT"] = u["second"] * u["_aut"]
    u["Bohr"] = 1e10 * 4 * math.pi * _eps0 * _hbar ** 2 / _me / _e ** 2
    u["Hartree"] = _me * _e ** 3 / 16 / math.pi ** 2 / _eps0 ** 2 / _hbar ** 2
    u["Ha"] = u["Hartree"]
    u["Rydberg"] = u["Ry"] = 0.5 * u["Hartree"]
    u["mol"] = _Nav
    u["kJ"] = 1000.0 / _e
    u["kcal"] = 4.184 * u["kJ"]
    u["J"] = 1.0 / _e
    u["C"] = 1.0 / _e
    u["s"] = u["second"]
    u["A"] = 1.0 / _e / u["second"]           # Ampere, as in ASE
    u["ms"] = 1e-3 * u["second"]
    u["us"] = 1e-6 * u["second"]
    u["ns"] = 1e-9 * u["second"]
    u["ps"] = 1e-12 * u["second"]
    u["kg"] = 1.0 / _amu
    return u


_UNITS = _ase_units()


def _factor(unit: str) -> float:
    if unit == "A":     # units.py:132-137
        raise Warning("The unit string 'A' specifies Ampere. For Angstrom, please use 'Ang' or 'Angstrom'.")
    try:
        return _UNITS[unit]
    except KeyError:
        raise AttributeError(f"unknown unit {unit!r}") from None


def _parse_unit(unit: Union[str, float]) -> float:
    """units.py:146-168: products and quotients of unit names, e.g. ``"kcal / mol"``; numbers pass through."""
    if not isinstance(unit, str):
        return unit
    conversion, divide = 1.0, False
    for part in re.split(r"(\W)", unit):
        if part == "/":
            divide = True
        elif part in ("", " "):
            pass
        else:
            p = _factor(part)
            if divide:
                conversion /= p
                divide = False
            else:
                conversion *= p
    return conversion


def convert_units(src_unit: Union[str, float], tgt_unit: Union[str, float]) -> float:
    """Factor that converts a quantity in ``src_unit`` to ``tgt_unit`` (units.py:184-186)."""
    return _parse_unit(src_unit) / _parse_unit(tgt_unit)

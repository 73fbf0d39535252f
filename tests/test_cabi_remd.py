"""CPU: the replica-exchange and per-system thermostat entry points of include/spk_b200.h are exported by the library and
bound by _lib with their launch counts; arguments are refused before any launch; thermostats that sample no canonical
ensemble, or act on ring polymers, refuse per-system temperatures."""
import ctypes

import pytest
import torch


def test_remd_entry_points_exported_and_bound():
    from schnetpack_b200 import _lib, build

    h = ctypes.CDLL(build.build())
    for name in ("spk_md_langevin_per_system", "spk_md_nhc_per_system", "spk_remd_exchange"):
        assert hasattr(h, name), name
        assert name in _lib.SIGNATURES
    sig = _lib.SIGNATURES
    # the per-system entry points are the scalar ones with idx_m / the kB T table added
    assert sig["spk_md_langevin_per_system"][:3] == [ctypes.c_void_p] * 3
    assert len(sig["spk_md_langevin_per_system"]) == len(sig["spk_md_langevin"]) + 1
    assert len(sig["spk_md_nhc_per_system"]) == len(sig["spk_md_nhc"]) + 1
    assert len(sig["spk_remd_exchange"]) == 20
    assert sig["spk_remd_exchange"][-2]._type_ is _lib.STRUCTS["spk_remd_buffers_t"]
    # decide + swap; per-system NHC: kinetic-energy partials, chains, scaling (one kernel when massive)
    assert _lib.LAUNCHES["spk_remd_exchange"] == 2
    assert _lib.LAUNCHES["spk_md_nhc_per_system"] == 3
    assert _lib.LAUNCHES.get("spk_md_langevin_per_system", 1) == 1
    table = _lib.STRUCTS["spk_remd_buffers_t"]
    n = _lib.CONSTANTS["SPK_REMD_MAX_BUFFERS"]
    assert [f for f, _ in table._fields_] == ["n_buffers", "per_atom", "width", "data"]
    assert all(t._length_ == n for _, t in table._fields_[1:])


def _exchange(**kw):
    from schnetpack_b200 import _lib

    buf = (ctypes.c_int64 * 64)()
    p = ctypes.addressof(buf)
    args = dict(energy=p, e_conv=1.0, temperature=p, kB=1.0, idx_m=None, sys_ptr=None, n_atoms=0, n_groups=2, n_rungs=3,
                seed=0, step=None, every=1, attempt=p, walker=p, attempted=p, accepted=p, decision=p, momenta=None,
                buffers=None, stream=None)
    args.update(kw)
    return _lib.lib().spk_remd_exchange(*args.values())


@pytest.mark.parametrize("bad", [dict(n_rungs=1), dict(n_groups=0), dict(every=0), dict(kB=0.0), dict(energy=None),
                                 dict(walker=None), dict(decision=None), dict(n_atoms=5)])
def test_remd_exchange_refuses_bad_arguments(bad):
    from schnetpack_b200 import _lib

    assert _exchange(**bad) == _lib.SPK_ERR_ARG


def test_remd_exchange_refuses_a_bad_buffer_table():
    from schnetpack_b200 import _lib

    table = _lib.STRUCTS["spk_remd_buffers_t"]()
    table.n_buffers = _lib.CONSTANTS["SPK_REMD_MAX_BUFFERS"] + 1
    assert _exchange(buffers=ctypes.byref(table)) == _lib.SPK_ERR_ARG
    table.n_buffers = 1                                  # data[0] NULL
    assert _exchange(buffers=ctypes.byref(table)) == _lib.SPK_ERR_ARG


def test_per_system_entry_points_need_their_table():
    from schnetpack_b200 import _lib

    h = _lib.lib()
    ctr = (ctypes.c_int64 * 2)()
    assert h.spk_md_langevin_per_system(None, None, None, 0, 0.5, 0.5, None, 0, ctypes.addressof(ctr), None) == \
        _lib.SPK_ERR_ARG
    params = _lib.NHCParams(3, 2, 3, 0, 0.0, (ctypes.c_double * 7)())
    x = ctypes.addressof(ctr)
    assert h.spk_md_nhc_per_system(None, None, None, None, 0, 1, ctypes.byref(params), None, x, x, x, x, 64, None) == \
        _lib.SPK_ERR_ARG


@pytest.mark.parametrize("make", [
    lambda M: M.BerendsenThermostat([300.0, 310.0], 10.0),
    lambda M: M.PILELocalThermostat([300.0, 310.0], 10.0),
    lambda M: M.TRPMDThermostat(torch.tensor([300.0, 310.0]), 0.5),
    lambda M: M.NHCRingPolymerThermostat([300.0], 10.0),
    lambda M: M.NHCBarostatIsotropic(1.0, [300.0, 310.0], 10.0),
    lambda M: M.PILEBarostat(1.0, [300.0, 310.0], 10.0),
])
def test_scalar_thermostats_refuse_per_system_temperatures(make):
    from schnetpack_b200 import md as M

    with pytest.raises(ValueError, match="temperature_bath must be one number"):
        make(M)


def test_per_system_thermostats_take_sequences_and_tensors():
    from schnetpack_b200 import md as M

    assert M.LangevinThermostat([300.0, 310.0], 10.0).temperature_bath == [300.0, 310.0]
    assert M.NHCThermostat(torch.tensor([300.0, 310.0]), 10.0).per_system
    assert not M.NHCThermostat(torch.tensor(300.0), 10.0).per_system
    assert not M.LangevinThermostat(300, 10.0).per_system
    from schnetpack_b200.exchange import ReplicaExchange

    for bad in (dict(n_temperatures=1, every_n_steps=1), dict(n_temperatures=2.5, every_n_steps=1),
                dict(n_temperatures=4, every_n_steps=0)):
        with pytest.raises(ValueError):
            ReplicaExchange(**bad)

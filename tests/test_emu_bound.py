"""The bound pass of the two-phase loop NW on the host SIMT emulator (CPU suite): every case of tests/bound_cases.py at emulator size
(a few hundred jobs per kernel and option set) through dada2b_test_raw_bounds / dada2b_test_bound against tests/bound_ref.py, and the
replay of syn2000_default's NW comparisons with the E_minmax each met.  The GPU suite runs the same at full size in
test_gpu_zz_bound.py."""
import os
import platform
import sys

import pytest

from oracle import port

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

pytestmark = [pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only"),
              pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle_port.so is not built")]


@pytest.fixture()
def emu(monkeypatch):
    import ctypes

    import build_emu
    import dada2_b200.api as api
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    h = ctypes.CDLL(lib)
    h.cuemu_launches.restype = ctypes.c_long
    h.cuemu_launches.argtypes = [ctypes.c_char_p]
    h.cuemu_reset_launches()
    yield h


def test_emu_bound_cases(emu):
    import dada2_b200.api as api
    from tests import bound_cases as BC
    for case in BC.all_cases("emu"):
        BC.run_case(api.Resident, case)
    for k in (b"k_raw_bounds", b"k_nwrow<", b"k_nwlane<", b"k_nwfwd<", b"k_gapless_loop"):
        assert emu.cuemu_launches(k) > 0, k


def test_emu_bound_replay_syn2000(emu):
    import dada2_b200.api as api
    from tests import bound_cases as BC
    tot = BC.replay(api.Resident, "syn2000_default")
    for which, (dropped, n) in tot.items():
        assert n > 1000 and dropped > 0.5 * n, (which, dropped, n)

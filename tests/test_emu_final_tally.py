"""The final pass's diagonal-list tally (dd_final.cu: k_ft_count / k_ft_scatter / k_final_tally) and round 0 through the two-phase
diagonal test, on the host SIMT emulator (tests/emu) -- CPU suite.  Every run returns the reference's full result
(tests/final_tally_cases.py), on one context, with DADA2B_LANE_MAX moving round 0 between the lane-group kernel and the
thread-per-pair kernels, and on sharded runs (ranks as threads, the emulator's in-process NCCL stand-in)."""
import os
import platform
import sys

import pytest

from tests import final_tally_cases as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))

pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture(scope="module")
def emu_lib():
    import build_emu
    return build_emu.build()


@pytest.fixture()
def emu(emu_lib, monkeypatch):
    import ctypes

    import dada2_b200.api as api
    monkeypatch.setattr(api, "_LIBPATH", emu_lib)
    monkeypatch.setattr(api, "_LIB", None)
    h = ctypes.CDLL(emu_lib)
    h.cuemu_launches.restype = ctypes.c_long
    h.cuemu_launches.argtypes = [ctypes.c_char_p]
    h.cuemu_reset_launches()
    yield h


@pytest.mark.parametrize("name", F.NAMES)
def test_emu_final_tally_matches_reference(emu, name):
    import dada2_b200
    F.run_case(name, dada2_b200.dada_uniques)
    assert emu.cuemu_launches(b"k_final_tally") > 0 and emu.cuemu_launches(b"k_ft_count") > 0


@pytest.mark.parametrize("lane_max", ["0", "32", "16384"])
@pytest.mark.parametrize("name", ["big_cluster", "indels_ragged"])
def test_emu_round0_kernels_by_lane_max(emu, monkeypatch, name, lane_max):
    """0: round 0's bound pass on the thread-per-pair row kernel (equal lengths) or the forward-carry kernel; 32: the same, with the
    later small rounds on the lane-group kernel; 16384 (the default): round 0 of these small samples in one lane-group launch."""
    import dada2_b200
    monkeypatch.setenv("DADA2B_LANE_MAX", lane_max)
    F.run_case(name, dada2_b200.dada_uniques)
    assert (emu.cuemu_launches(b"k_nwlane<") > 0) == (lane_max != "0")


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", F.NAMES)
def test_emu_final_tally_sharded(emu, world, name):
    """Every rank tallies the diagonal raws it owns; the all-reduced sums and nsubs are the reference's on every rank."""
    from tests.test_emu_parity import _run_sharded
    seqs, ab, q, opts = F.sample(name)
    _run_sharded(world, name, case=(seqs, ab, None, q, opts))

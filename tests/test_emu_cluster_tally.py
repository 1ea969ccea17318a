"""The per-cluster tallies and $map of dada()'s output (dd_final.cu: k_cluster_tally) and repeated runs of one resident sample,
on the host SIMT emulator (tests/emu) -- CPU suite.  Cases: tests/cluster_tally_cases.py."""
import os
import platform
import sys

import pytest

from tests import cluster_tally_cases as C
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


@pytest.mark.parametrize("name", C.GOLDEN_NAMES)
def test_emu_cluster_tally_goldens(emu, name):
    import dada2_b200
    C.run_golden(name, dada2_b200.dada_uniques)
    assert emu.cuemu_launches(b"k_cluster_tally") > 0


@pytest.mark.parametrize("name", ["many_clusters", "omegaC"])
def test_emu_cluster_tally_samples(emu, name):
    import dada2_b200
    C.run_sample(name, dada2_b200.dada_uniques)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("name", ["many_clusters", "omegaC"])
def test_emu_cluster_tally_sharded(emu, world, name):
    """Every rank counts its own raws; the all-reduced tallies and $map are the reference's on every rank."""
    from tests.test_emu_parity import _run_sharded
    seqs, ab, q, opts = F.sample(name)
    _run_sharded(world, name, case=(seqs, ab, None, q, opts))


def test_emu_repeated_runs_on_one_context(emu, monkeypatch):
    C.run_repeated(monkeypatch)

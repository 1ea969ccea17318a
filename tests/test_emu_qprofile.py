"""The quality profile's kernels (dd_qprofile.cu) and plotQualityProfile / plotComplexity on the host SIMT emulator --
CPU suite; the same cases as tests/test_gpu_zz_qprofile.py, and again with DADA2B_SMS=1 so that one block walks many
read chunks and cycle tiles."""
import os
import platform
import sys

import numpy as np
import pytest

from tests import qprofile_cases as G
from tests import qprofile_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.filter as fl
    import dada2_b200.qc as qc
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(fl, "_BOUND", False)
    monkeypatch.setattr(qc, "_BOUND", False)
    yield lib


def test_emu_qprofile_cases(emu, tmp_path):
    G.check_profiles(str(tmp_path))


def test_emu_qprofile_complexity(emu, tmp_path):
    G.check_complexity(str(tmp_path))


def test_emu_qprofile_edges_and_refusals(emu, tmp_path):
    G.check_edges_and_refusals(str(tmp_path))


def test_emu_qprofile_one_sm(emu, tmp_path, monkeypatch):
    """DADA2B_SMS=1: four blocks walk every (chunk, tile) item of 20 000 ragged reads over 9 tiles."""
    from dada2_b200 import qc
    monkeypatch.setenv("DADA2B_SMS", "1")
    rng = np.random.default_rng(3)
    lens = rng.integers(0, 9 * G.TILE, 20000)
    off = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    qual = rng.choice(np.array([2, 12, 23, 37, 93], np.uint8), int(off[-1]), p=[0.05, 0.05, 0.1, 0.75, 0.05])
    got, st = qc.quality_tally(off, qual)
    want = R.tally_packed(off, qual)
    assert np.array_equal(got, want)
    G.check_profiles(str(tmp_path))

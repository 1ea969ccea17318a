"""Species assignment (dd_species.cu) on the host SIMT emulator -- CPU suite; the same checks as
tests/test_gpu_zz_species.py without the large database: hit lists and assignments equal to the restatement on the man
page's example and on the synthetic edge set, unchanged with a one-record hit buffer, offset-0 anchors, small batches
and a reused database; and every refusal."""
import os
import platform
import sys

import pytest

from tests import species_cases as G

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.species as sp
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(sp, "_BOUND", False)
    yield lib


def test_emu_species_example(emu):
    G.run_example()


def test_emu_species_synthetic(emu, monkeypatch):
    G.run_synthetic(monkeypatch)


def test_emu_species_refusals(emu):
    G.check_refusals()

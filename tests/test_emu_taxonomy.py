"""Taxonomic classification (dd_taxonomy.cu) on the host SIMT emulator -- CPU suite; the same checks as
tests/test_gpu_zz_taxonomy.py on the example training set: bit-exact against the restatement, the table under the
1-ulp rule, the logp hook, explicit uniforms, resident reuse, forced chunking and every refusal."""
import os
import platform
import sys

import pytest

from tests import taxonomy_cases as G

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.taxonomy as tx
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(tx, "_BOUND", False)
    yield lib


def test_emu_taxonomy_exact(emu):
    db, lgk, nbad = G.run_all()
    print("1-ulp table entries: %d of %d" % (nbad, lgk.size))


def test_emu_taxonomy_chunking(emu, monkeypatch):
    G.check_chunking(monkeypatch, seqs_n=2)


def test_emu_taxonomy_refusals(emu):
    G.check_refusals()

"""Primer removal (dd_primer.cu) on the host SIMT emulator -- CPU suite; the same assertions as
tests/test_gpu_zz_primer.py on every golden case, through the hit hook, over files, and on every refusal."""
import os
import platform
import sys

import pytest

from tests import primer_cases as G

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.primer as pm
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(pm, "_BOUND", False)
    yield lib


def test_emu_primer_golden_cases_and_hits(emu):
    from dada2_b200 import primer as pm
    g = G.load_golden()
    for case in G.cases():
        G.check_case(case, G.run_product(case, pm.remove_primers_reads), G.want_from_golden(g, case))
        G.check_hits(case, pm.test_primer_hits, g[case["name"] + "/hits"])


def test_emu_primer_files_and_errors(emu, tmp_path):
    G.check_files(str(tmp_path))
    G.check_errors()

"""The read filter's kernels (dd_filter.cu) on the host SIMT emulator -- CPU suite; the same assertions as
tests/test_gpu_zz_filter.py on every golden case and through the stage hook."""
import math
import os
import platform
import sys

import numpy as np
import pytest

from tests import filter_cases as G
from tests import filter_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.filter as fl
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(fl, "_BOUND", False)
    yield lib


def test_emu_filter_golden_cases(emu):
    from dada2_b200 import filter as fl
    g = G.load_golden()
    for case in G.all_cases():
        G.check_case(case, G.run_product(case, fl.filter_reads), G.want_from_golden(g, case))


def test_emu_filter_stage_hook(emu):
    from dada2_b200 import filter as fl
    for case in G.single_cases():
        G.check_stages(case, fl.test_filter_stages)


def test_emu_filter_errors_and_helpers(emu):
    G.check_errors_and_helpers()

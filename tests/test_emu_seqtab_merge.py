"""mergeSequenceTables' kernels (dd_seqtab.cu) on the host SIMT emulator -- CPU suite: every hand case against its
literal expectation and the restatement, and seeded multi-run merges (tryRC on and off, shared sample names) against
the restatement."""
import os
import platform
import sys

import numpy as np
import pytest

from tests import seqtab_merge_cases as G

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.seqtab as st
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(st, "_BOUND", False)
    yield lib


def test_emu_seqtab_merge_hand_cases(emu):
    G.check_hand()


@pytest.mark.parametrize("tryRC", [False, True])
def test_emu_seqtab_merge_seeded(emu, tryRC):
    runs = G.make_runs(11, nruns=4, nsamp=12, pool=400, per_run=150)
    G.check_seeded(runs, tryRC=tryRC)
    G.check_seeded(runs, tryRC=tryRC, orderBy="nsamples")


def test_emu_seqtab_merge_shared_samples(emu):
    """Sample names repeated across runs: those tables add with atomics, and runs in reverse orientation collapse."""
    runs = G.make_runs(12, nruns=3, nsamp=10, pool=300, per_run=120, rc_every=2, shared_frac=0.5)
    got = G.check_seeded(runs, tryRC=True, repeats="sum", orderBy=None)
    assert len(got[2]) < 30


def test_emu_seqtab_merge_stats(emu):
    from dada2_b200 import seqtab
    mats = [np.array([[1, 2]], np.int32), np.array([[3]], np.int32)]
    mat, src, st = seqtab.merge_columns(mats, [[G.S1, "GTTT"], ["TTTT"]], [0, 1], 2, tryRC=True, order_by=0)
    assert mat.tolist() == [[3, 0], [0, 3]] and src.tolist() == [0, 2] and st["n_rc"] == 1
    mat, src, st = seqtab.merge_columns(mats, [[G.S1, "GTTT"], ["TTTT"]], [0, 1], 2, tryRC=False, order_by=0)
    assert mat.tolist() == [[1, 2, 0], [0, 0, 3]] and src.tolist() == [0, 1, 2] and st["n_rc"] == 0
    assert st["gpu_launches"] > 0 and st["h2d_bytes"] > 0

"""collapseNoMismatch's kernels (dd_collapse.cu) on the host SIMT emulator -- CPU suite; the same assertions as
tests/test_gpu_zz_collapse.py on the golden tables and on every golden pair."""
import os
import platform
import sys

import numpy as np
import pytest

from tests import collapse_cases as G
from tests import collapse_ref as R

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


def _hook(seqs, pq, pr, m, vec, band):
    from dada2_b200 import seqtab
    return seqtab.test_collapse_pairs(seqs, pq, pr, minOverlap=m, vec=vec, band=band)


def test_emu_collapse_golden_tables(emu):
    from dada2_b200 import seqtab
    G.check_tables(seqtab.collapseNoMismatch)


def test_emu_collapse_pairs_golden(emu):
    G.check_pairs(_hook)


def test_emu_collapse_corners(emu):
    from dada2_b200 import Dada2bError, seqtab
    rng = np.random.default_rng(5)
    B = "".join("ACGT"[i] for i in rng.integers(0, 4, 60))
    # a query that matches two kept sequences goes to the first one kept; one shorter than minOverlap is screened exactly
    seqs = [B, B[2:], B[:-4], B[10:25], B[11:25], "ACGT" * 5]
    rep, st = seqtab.collapse_reps(seqs, return_stats=True)
    assert rep.tolist() == [0, 0, 0, 0, 0, 5]
    want = sum(R.screen(seqs[j], seqs[i], 20) for j in range(len(seqs)) for i in range(j))
    assert st["n_candidates"] == want == 10 and st["n_aligned"] + st["n_filtered"] == st["n_candidates"]
    ham = [[R.port_nwhamming(a, b) for b in seqs] for a in seqs]
    assert seqtab.nwhamming(seqs, [seqs[0]] * len(seqs), vec=True).tolist() == [h[0] for h in ham]
    assert seqtab.nwhamming(B, B[:30] + "A" + B[31:]) == R.port_nwhamming(B, B[:30] + "A" + B[31:], vec=False)
    with pytest.raises(Dada2bError, match="A/C/G/T"):
        seqtab.collapse_reps(["ACGTN" * 5, "ACGTA" * 5])
    with pytest.raises(Dada2bError, match="16-bit"):
        seqtab.collapse_reps(["A" * 7000, "A" * 6999])
    mat, cols, rows = seqtab.makeSequenceTable({"a": {B: 3, B[2:]: 5}, "b": {B[2:]: 1, seqs[5]: 5}})
    assert cols == [B[2:], seqs[5], B] and rows == ["a", "b"] and mat.tolist() == [[5, 0, 3], [1, 5, 0]]
    m, c = seqtab.collapseNoMismatch(mat, cols)
    assert c == [B[2:], seqs[5]] and m.tolist() == [[8, 0], [1, 5]]

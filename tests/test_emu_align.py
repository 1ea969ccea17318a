"""nwalign's kernel (dd_align.cu) and isShiftDenovo's pipeline (dd_collapse.cu) on the host SIMT emulator -- CPU suite:
every nwalign golden in every mode, every shift golden and the stage hook on every golden pair, and the corners of both
functions' argument rules."""
import os
import platform
import sys

import numpy as np
import pytest

from tests import nwalign_cases as N
from tests import shift_cases as K

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    yield lib


def test_emu_nwalign_golden(emu):
    from dada2_b200 import align
    N.check(align.nwalign, align.eval_counts)


def test_emu_shift_golden(emu):
    from dada2_b200 import isShiftDenovo
    K.check_flags(isShiftDenovo)


def test_emu_shift_pairs_golden(emu):
    from dada2_b200 import bimera
    K.check_pairs(lambda s, q, p, m: bimera.test_shift_pairs(s, q, p, minOverlap=m))


def test_emu_shift_stats_reconcile(emu):
    from dada2_b200 import bimera
    g = K.load()
    seqs, ab = K.case(g, "synthetic")
    for m in (0, 20):
        flag, st = bimera.shift_flags(seqs, ab, minOverlap=m, return_stats=True)
        assert np.array_equal(flag.astype(bool), g[K.flag_key("synthetic", m)])
        assert st["n_candidates"] == st["n_filtered"] + st["n_aligned"] == st["n_screened"] - st["n_equal"]
        assert st["n_flagged"] == int(flag.sum())
        if m == 0:
            assert st["n_screened"] == len(seqs) * (len(seqs) - 1) // 2
            assert st["n_candidates"] == len(g["synthetic_pq"])


def test_emu_nwalign_corners(emu, capsys):
    from dada2_b200 import Dada2bError, nwalign, seqtab
    a, b = "ACGTTACGGA" * 4, "CGTTACGGAT" * 4
    assert nwalign([], []) == []
    assert nwalign(a, [b, a]) == [nwalign(a, b), nwalign(a, a)]               # a one-element side is recycled
    assert nwalign("", "ACG") == ("---", "ACG") and nwalign("AC", "") == ("AC", "--") and nwalign("", "") == ("", "")
    with pytest.raises(Dada2bError, match="only A/C/G/T"):
        nwalign(a, "ACGTN")
    with pytest.raises(Dada2bError, match="only A/C/G/T"):
        nwalign(a, "acgt")                                                     # C_isACGT: upper case only
    with pytest.raises(Dada2bError, match="Homopolymer gap penalties are not implemented"):
        nwalign(a, b, vec=True, homo_gap=-3)
    with pytest.raises(Dada2bError, match="A/C/G/T"):
        nwalign(a, "ACGTN", vec=True)
    capsys.readouterr()
    got = nwalign([a, a], [b, b], endsfree=False, homo_gap=-3)
    err = capsys.readouterr().err
    assert err.count("A separate homopolymer gap penalty isn't implemented when endsfree=FALSE") == 1
    assert got == nwalign([a, a], [b, b], endsfree=False)
    # the int16 bound: ends-free by the longest sequence, global by len1 + len2 + 1
    with pytest.raises(Dada2bError, match="16-bit"):
        nwalign("A" * 7000, "A" * 6999, vec=True)
    with pytest.raises(Dada2bError, match="16-bit"):
        nwalign("A" * 2100, "A" * 2100, vec=True, endsfree=False)
    assert nwalign("A" * 2000, "A" * 2000, vec=True, endsfree=False) == ("A" * 2000, "A" * 2000)
    with pytest.raises(Dada2bError, match="maximum allowed string length"):
        nwalign("A" * 9999, "A")
    # nwhamming's pass-through of nwalign's arguments
    assert seqtab.nwhamming(a, b, endsfree=False) == int(np.sum(seqtab.nwhamming([a], [b], endsfree=False)))
    assert seqtab.nwhamming("", a) == 0


def test_emu_shift_corners(emu, capsys):
    from dada2_b200 import Dada2bError, isShiftDenovo
    rng = np.random.default_rng(2)
    B = "".join("ACGT"[i] for i in rng.integers(0, 4, 90))
    S = B[4:] + "ACGT"
    assert isShiftDenovo({}).tolist() == []
    assert isShiftDenovo({B: 10, S: 3}).tolist() == [False, True]
    assert isShiftDenovo({B: 10, S: 3}, flagSubseqs=True).tolist() == [False, True]
    assert isShiftDenovo({B: 10, S: 10}).tolist() == [False, False]            # equal abundances never pair
    assert isShiftDenovo({B: 10, S: 3}, minOverlap=90).tolist() == [False, False]
    # "" is never flagged and flags nothing; a non-A/C/G/T sequence errors only when it has a partner of other abundance
    assert isShiftDenovo({B: 10, S: 3, "": 50}).tolist() == [False, True, False]
    with pytest.raises(Dada2bError, match="only A/C/G/T"):
        isShiftDenovo({B: 10, S: 3, "ACGN" * 10: 10})                           # S (abundance 3) is a partner
    with pytest.raises(Dada2bError, match="only A/C/G/T"):
        isShiftDenovo({B: 10, S: 3, "ACGN" * 10: 7})
    assert isShiftDenovo({"ACGN" * 10: 7}).tolist() == [False]
    # the other input forms; a merger's duplicates are summed and every copy gets the flag
    assert isShiftDenovo({"denoised": {B: 10, S: 3}}).tolist() == [False, True]
    assert isShiftDenovo({"uniques": [B, S], "abundances": [10, 3]}).tolist() == [False, True]
    mg = {"sequence": [S, B, S, ""], "abundance": [2, 10, 2, 40], "forward": [1, 2, 1, 3]}
    assert isShiftDenovo(mg).tolist() == [True, False, True, False]
    mat = np.array([[1, 9], [2, 1]], np.int32)
    assert isShiftDenovo((mat, [S, B])).tolist() == [True, False]
    capsys.readouterr()
    isShiftDenovo({B: 10, S: 3, B[:50]: 10}, verbose=True)
    assert capsys.readouterr().out.count('"No possible parents."') == 2

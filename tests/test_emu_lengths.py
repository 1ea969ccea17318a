"""The length-driven layout switches of mergePairs, bimera detection, collapseNoMismatch and derep on the host SIMT
emulator -- CPU suite.  Each switch is crossed at a length the emulator finishes in seconds: a case just below and one
just above a threshold computed from the host code's own formula (tests/length_cases.py), each side checked against the
CPU oracle, and the kernel that ran on each side asserted through the emulator's launch counter or the case's layout
class.  tests/test_gpu_zz_lengths.py runs the same switches at real amplicon lengths on the GPU."""
import ctypes
import os
import platform
import sys

import numpy as np
import pytest

from tests import length_cases as LC

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")

EMU_BIM_SCORES = dict(match=5, mismatch=-40, gap_p=-8)      # puts the 16-bit kernel's headroom at about 200 nt
EMU_VEC_SCORES = dict(match=5, mismatch=-100, gap=-100)     # puts the vectorized aligner's limit at about 330 nt


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.bimera as bm
    import dada2_b200.derep as dr
    import dada2_b200.merge as mg
    import dada2_b200.seqtab as st
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    for m in (bm, dr, mg, st):
        monkeypatch.setattr(m, "_BOUND", False)
    h = ctypes.CDLL(lib)
    h.cuemu_launches.restype = ctypes.c_long
    h.cuemu_launches.argtypes = [ctypes.c_char_p]
    yield h


def launches(h, names):
    return {n: h.cuemu_launches(n.encode()) for n in names}


def check_merge(pool, s1, s2, prefer, **o):
    from dada2_b200 import merge
    from oracle import port
    got = merge.merge_align(pool, s1, s2, prefer, **o)
    for x in range(len(s1)):
        w = port.merge_pair(pool[s1[x]], pool[s2[x]], prefer=int(prefer[x]), **o)
        g = (int(got["nmatch"][x]), int(got["nmismatch"][x]), int(got["nindel"][x]), got["sequence"][x])
        assert g == (w["nmatch"], w["nmismatch"], w["nindel"], w["sequence"]), (o, x, g)


@pytest.mark.parametrize("band", [-1, 16])
def test_emu_merge_scratch_switch(emu, band):
    """k_merge_pairs with its move matrix in shared memory (batch maxlen one below the switch) and in global scratch
    (at the switch), unbanded and with band 16 over equally long reads."""
    from dada2_b200 import Dada2bError, merge
    sw = LC.scratch_switch(band)
    sides = []
    for maxlen in (sw - 1, sw):
        if band < 0:
            pool, s1, s2, pref = LC.merge_batch_at(maxlen, 3, seed=maxlen)
        else:                                       # overlaps within the band; a 20 nt overlap leaves it, as in the reference
            pool, s1, s2, pref = LC.merge_batch_at(maxlen, 2, seed=maxlen, overlap=(maxlen - 10, maxlen), equal=True)
            p2 = LC.merge_batch_at(maxlen, 1, seed=maxlen, overlap=(20, 20), equal=True)
            with pytest.raises(Dada2bError, match="N-W Align out of range"):
                merge.merge_align(*p2, band=band)
        lens = [len(s) for s in pool]
        sides.append(LC.nw_layout(max(lens), min(lens), band))
        opts = (dict(band=band), dict(band=band, mismatch=-8, gap_p=-8, trim_overhang=True))
        for o in opts:
            check_merge(pool, s1, s2, pref, **o)
    assert sides == ["smem", "global"], sides


def test_emu_bimera_int16_headroom(emu, monkeypatch):
    """k_bimfwd16 takes the batch one base below its int16 headroom and hands it to k_bimfwd one base above."""
    from dada2_b200 import bimera
    from oracle import port
    monkeypatch.setenv("DADA2B_BIMFWD", "2")
    top = LC.bim16_maxlen(EMU_BIM_SCORES["match"], EMU_BIM_SCORES["mismatch"], EMU_BIM_SCORES["gap_p"])
    names = ("k_bimfwd16<", "k_bimfwd<", "k_bim_align")
    for maxlen, want in ((top, "k_bimfwd16"), (top + 1, "k_bimfwd")):
        assert LC.bim_route(maxlen, maxlen, 16, EMU_BIM_SCORES["match"], EMU_BIM_SCORES["mismatch"], EMU_BIM_SCORES["gap_p"]) == want
        seqs, q, p = LC.bimera_pairs_at(maxlen, 0, 2, seed=maxlen)
        n0 = launches(emu, names)
        got = bimera.test_bimera_pairs(seqs, q, p, allow_one_off=True, **EMU_BIM_SCORES)
        n1 = launches(emu, names)
        ran16 = n1["k_bimfwd16<"] - n0["k_bimfwd16<"]
        assert ran16 == (want == "k_bimfwd16") and n1["k_bimfwd<"] - n0["k_bimfwd<"] == 1, (maxlen, n0, n1)
        for n, (a, b) in enumerate(zip(q, p)):
            r = port.bimera_pair(seqs[a], seqs[b], allow_one_off=True, **EMU_BIM_SCORES)
            assert list(got[n]) == [r["left"], r["right"], r["left_oo"], r["right_oo"], r["ham"]], (maxlen, n)


def test_emu_bimera_slot_classes(emu, monkeypatch):
    """Length spreads that put the batch's slots_needed on each side of every class bound of pick16 / pick: each side
    runs k_bimfwd16 in its own instantiation; past the last class everything goes to k_bim_align."""
    from dada2_b200 import bimera
    from oracle import port
    monkeypatch.setenv("DADA2B_BIMFWD", "2")
    names = ("k_bimfwd16<", "k_bimfwd<", "k_bim_align")
    L = 250
    for bound, below, above in LC.slot_spreads(16):
        cls = [LC.bim_class(LC.bim_slots(L, L - d, 16)) for d in (below, above)]
        assert cls[0][0] == bound and (cls[1] is None or cls[1][0] > bound), (bound, cls)
        for d in (below, above):
            route = LC.bim_route(L, L - d, 16)
            seqs, q, p = LC.bimera_pairs_at(L, d, 2, seed=bound + d)
            n0 = launches(emu, names)
            got = bimera.test_bimera_pairs(seqs, q, p, allow_one_off=True)
            n1 = launches(emu, names)
            assert n1["k_bimfwd16<"] - n0["k_bimfwd16<"] == (route == "k_bimfwd16"), (bound, d, route)
            if route == "k_bim_align":
                assert n1["k_bimfwd<"] == n0["k_bimfwd<"] and n1["k_bim_align"] - n0["k_bim_align"] == 1
            for n, (a, b) in enumerate(zip(q, p)):
                r = port.bimera_pair(seqs[a], seqs[b], allow_one_off=True)
                assert list(got[n]) == [r["left"], r["right"], r["left_oo"], r["right_oo"], r["ham"]], (bound, d, n)
    assert LC.bim_route(L, L - LC.slot_spreads(16)[-1][2], 16) == "k_bim_align"


def test_emu_collapse_vec_limit(emu):
    """vec=TRUE at the largest maxlen the int16 guard accepts (aligned, against the CPU port) and the smallest it refuses;
    vec=FALSE has no such limit."""
    from dada2_b200 import Dada2bError, seqtab
    from tests import collapse_ref as R
    sc = EMU_VEC_SCORES
    top = LC.vec_maxlen(sc["match"], sc["mismatch"], sc["gap"])
    assert LC.vec_fits(top, **sc) and not LC.vec_fits(top + 1, **sc)
    for maxlen in (top, top + 1):
        seqs, q, r = LC.collapse_pairs_at(maxlen, 5, seed=maxlen)
        for vec, band in ((True, -1), (True, 16), (False, -1)):
            if vec and maxlen > top:
                with pytest.raises(Dada2bError, match=LC.VEC_REFUSAL):
                    seqtab.test_collapse_pairs(seqs, q, r, minOverlap=20, vec=vec, band=band, **sc)
                with pytest.raises(Dada2bError, match=LC.VEC_REFUSAL):
                    seqtab.collapse_reps(seqs, vec=vec, band=band, **sc)
                continue
            out = seqtab.test_collapse_pairs(seqs, q, r, minOverlap=20, vec=vec, band=band, **sc)
            for x in range(len(q)):
                a, b = seqs[q[x]], seqs[r[x]]
                assert out[x, 0] == R.screen(a, b, 20), (maxlen, vec, band, x)
                assert out[x, 2] == R.port_nwhamming(a, b, vec=vec, band=band, **sc), (maxlen, vec, band, x)
                assert out[x, 1] == R.overlap_filter(a, b, sc["match"], sc["mismatch"], band), (maxlen, vec, band, x)
            assert (out[:, 2] == 0).any() and (out[:, 2] > 0).any()


def test_emu_derep_key_word_boundaries(emu):
    """Reads whose length ends a key word, starts the next one, or sits one short of it; the longest accepted length;
    the first refused one, with the reference's message."""
    from dada2_b200 import Dada2bError, derep
    from oracle import derep as O
    from tests import derep_cases as D
    kw = [LC.derep_key_words(L) for L in (15, 16, 17, 31, 32, 33)]
    assert kw == [1, 1, 2, 2, 2, 3]
    for L in LC.DEREP_LENGTHS:
        s, q = LC.derep_reads(L, 6 if L < 1000 else 3, 60 if L < 1000 else 20, seed=L, qmax=93)
        for n in (1000000, 7):
            D.assert_same(derep.derep_reads(s, q, n=n), O.derep_reads(s, q, n=n), "L=%d n=%d" % (L, n))
    s, q = LC.derep_reads(LC.SEQLEN, 2, 4, seed=1)
    with pytest.raises(Dada2bError, match=LC.DEREP_REFUSAL):
        derep.derep_reads(s, q)

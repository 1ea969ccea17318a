"""mergePairs over whole samples (dd_pairs.cu + dd_merge.cu) on the host SIMT emulator against the restatement
(tests/paired_ref.py), field by field -- CPU suite; tests/test_gpu_zz_paired.py runs the same comparisons on the H100 at
real amplicon lengths."""
import os
import platform
import subprocess
import sys

import numpy as np
import pytest

from tests import paired_cases as P
from tests import paired_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "emu"))
pytestmark = pytest.mark.skipif(platform.machine() != "x86_64", reason="the emulator's fiber switch is x86-64 only")


@pytest.fixture()
def emu(monkeypatch):
    import build_emu
    import dada2_b200.api as api
    import dada2_b200.paired as pp
    lib = build_emu.build()
    monkeypatch.setattr(api, "_LIBPATH", lib)
    monkeypatch.setattr(api, "_LIB", None)
    monkeypatch.setattr(pp, "_BOUND", False)
    yield lib


HAND = [("hand", P.hand_sample, {}), ("hand_rejects", P.hand_sample, dict(returnRejects=True)),
        ("hand_mm1", P.hand_sample, dict(maxMismatch=1)),
        ("hand_concat", P.hand_sample, dict(justConcatenate=True, propagateCol=("n0", "birth_ham", "not_a_column"))),
        ("overhang", P.overhang_sample, dict(maxMismatch=1, returnRejects=True)),
        ("overhang_trim", P.overhang_sample, dict(maxMismatch=1, trimOverhang=True)),
        ("hand_scores", P.hand_sample, dict(returnRejects=True, match=2, mismatch=-3, gap=-5, homo_gap=-2))]


@pytest.mark.parametrize("name,case,kw", HAND, ids=[h[0] for h in HAND])
def test_emu_hand_cases_match_restatement(emu, name, case, kw):
    from dada2_b200 import mergePairs
    got = mergePairs(*case(), **kw)
    R.assert_same(got, R.merge_sample(*case(), **kw), name)


def test_emu_empty_sample_duplicates_and_shapes(emu, capsys):
    from dada2_b200 import mergePairs
    dF, rF, dR, rR = P.hand_sample()
    eF, erF, eR, erR = P.empty_sample()
    got = mergePairs({"a": dF, "b": eF}, {"a": rF, "b": erF}, {"a": dR, "b": eR}, {"a": rR, "b": erR}, verbose=True, returnRejects=True)
    assert list(got) == ["a", "b"]
    R.assert_same(got["b"], R.merge_sample(eF, erF, eR, erR), "empty")
    err = capsys.readouterr().err
    assert "5 paired-reads (in 2 unique pairings) successfully merged out of 7 (in 3 pairings) input." in err
    assert "No paired-reads (in ZERO unique pairings) successfully merged out of 3 pairings) input." in err
    lst = mergePairs([dF, dF], [rF, rF], [dR, dR], [rR, rR])
    assert isinstance(lst, list) and len(lst) == 2
    one = mergePairs([dF], [rF], [dR], [rR])
    assert isinstance(one, dict) and one["forward"].tolist() == [2, 1]
    # the same merged sequence from two pairings: R's message
    dF2 = P.dada_obj([P.AMP[:60], P.AMP[:61]], [5, 1], [1, 2, 1, None])
    capsys.readouterr()
    mergePairs(dF2, rF, dR, rR)
    assert "Duplicate sequences in merged output." in capsys.readouterr().err


def test_emu_non_corresponding_and_non_acgt(emu):
    from dada2_b200 import mergePairs, Dada2bError
    dF, rF, dR, rR = P.hand_sample()
    for c in [(dF, P.derep_obj(4, rF["map"][:-1]), dR, rR), (P.dada_obj(["ACGT"], [1], [1, 1, 1]), rF, dR, rR),
              (dF, rF, dR, P.derep_obj(3, [1] * 9)), (dF, P.derep_obj(4, [None] * 9), dR, rR)]:
        with pytest.raises(Dada2bError, match="Non-corresponding derep-class and dada-class objects."):
            mergePairs(*c)
    bad = P.dada_obj([P.AMP[:60], P.AMP[:59] + "N"], [5, 1], [1, 2, 1, None])
    with pytest.raises(Dada2bError, match="A/C/G/T"):
        mergePairs(bad, rF, dR, rR)


def _multi(sets, monkeypatch, batch, **kw):
    from dada2_b200 import mergePairs
    if batch is None:
        monkeypatch.delenv("DADA2B_PAIRS_BATCH", raising=False)
    else:
        monkeypatch.setenv("DADA2B_PAIRS_BATCH", str(batch))
    dFs, rFs, dRs, rRs = [list(x) for x in zip(*sets)]
    got, st = mergePairs(dFs, rFs, dRs, rRs, return_stats=True, **kw)
    want = [R.merge_sample(*c, **kw) for c in sets]
    for i, (g, w) in enumerate(zip(got, want)):
        R.assert_same(g, w, "sample %d" % i)
    return st


@pytest.mark.parametrize("batch", [None, 700, 1], ids=["one_batch", "batch700", "batch1"])
def test_emu_synthetic_samples_and_batches(emu, monkeypatch, batch):
    sets = P.synth_set(5, 300, seed=7, lenlo=100, lenhi=150, readlen=80)
    sets.append(P.synth_set(1, 1500, seed=8, lenlo=100, lenhi=150, readlen=80)[0])      # larger than the 700-read batch: alone
    st = _multi(sets, monkeypatch, batch, returnRejects=True, propagateCol=("n0",))
    allm = [R.merge_sample(*c, returnRejects=True) for c in sets]
    assert st["n_aligned"] == R.distinct_triples([c[0] for c in sets], [c[2] for c in sets], allm)
    assert st["n_pairings"] == sum(len(m["forward"]) for m in allm) and st["n_reads"] == sum(len(c[1]["map"]) for c in sets)
    assert st["n_batches"] == {None: 1, 700: 4, 1: 6}[batch]


def test_emu_synthetic_options(emu, monkeypatch):
    sets = P.synth_set(3, 200, seed=11, lenlo=100, lenhi=150, readlen=80)
    _multi(sets, monkeypatch, 250, maxMismatch=1, trimOverhang=True, returnRejects=True)
    st = _multi(sets, monkeypatch, 250, justConcatenate=True)
    assert st["n_aligned"] == 0


SCRIPT = """
import sys
sys.path.insert(0, %r)
import dada2_b200.api as api
api._LIBPATH = %r; api._LIB = None
from dada2_b200 import mergePairs
from tests import paired_cases as P, paired_ref as R
sets = [P.hand_sample(), P.overhang_sample(), P.empty_sample()] + P.synth_set(3, 150, seed=5, lenlo=100, lenhi=140, readlen=80)
for kw in (dict(returnRejects=True), dict(justConcatenate=True, maxMismatch=1)):
    got = mergePairs(*[list(x) for x in zip(*sets)], **kw)
    for c, g in zip(sets, got):
        R.assert_same(g, R.merge_sample(*c, **kw))
print('ASAN RUN OK')
"""


def test_emu_paired_kernels_are_memory_clean_under_asan(monkeypatch):
    from tests.test_emu_asan import _preload
    asan = _preload()
    if asan is None:
        pytest.skip("libasan not found")
    import build_emu
    lib = build_emu.build(asan=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1", DADA2B_PAIRS_BATCH="200")
    out = subprocess.run([sys.executable, "-c", SCRIPT % (ROOT, lib)], env=env, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert "AddressSanitizer" not in out.stderr, out.stderr[-4000:]
    assert out.returncode == 0 and "ASAN RUN OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]

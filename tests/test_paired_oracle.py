"""mergePairs' restatement (tests/paired_ref.py) against hand-worked tables, and mergePairs' argument checks, which all run
before any native call.  CPU suite."""
import numpy as np
import pytest

from tests import paired_cases as P
from tests import paired_ref as R

A = P.AMP
NA = R.NA


def _cols(m):
    return {k: (list(v) if isinstance(v, list) else v.tolist()) for k, v in m.items()}


def test_hand_sample_na_maps_and_tie_order():
    # reads -> (rF, rR): (1,1) (2,1) (1,2) NA (1,1) NA (2,1) (1,2) (2,1): (2,1) x3 first, then the tie (1,1) / (1,2) by first read
    m = R.merge_sample(*P.hand_sample(), returnRejects=True)
    assert _cols(m) == {"sequence": [P.sub(A, 5), A, ""], "abundance": [3, 2, 2], "forward": [2, 1, 1], "reverse": [1, 1, 2],
                        "nmatch": [20, 20, 0], "nmismatch": [0, 0, 0], "nindel": [0, 0, 0], "prefer": [2, 1, 2],
                        "accept": [True, True, False]}
    m = R.merge_sample(*P.hand_sample())
    assert m["forward"].tolist() == [2, 1] and m["sequence"] == [P.sub(A, 5), A]


def test_max_mismatch_one():
    m = R.merge_sample(*P.hand_sample(), maxMismatch=1)
    assert m["nmatch"].tolist() == [20, 20, 19] and m["nmismatch"].tolist() == [0, 0, 1] and m["accept"].all()
    assert m["sequence"][2] == P.sub(A, 50)                              # prefer 2: the reverse read's base


def test_trim_overhang():
    m = R.merge_sample(*P.overhang_sample(), maxMismatch=1)
    assert m["sequence"] == [A[:80], P.sub(A, 40)[:80]] and m["nmatch"].tolist() == [60, 59] and m["prefer"].tolist() == [1, 2]
    m = R.merge_sample(*P.overhang_sample(), maxMismatch=1, trimOverhang=True)
    assert m["sequence"] == [A[10:70], P.sub(A, 40)[10:70]]


def test_just_concatenate_and_propagate_col():
    m = R.merge_sample(*P.hand_sample(), justConcatenate=True, propagateCol=("n0", "birth_ham", "not_a_column"))
    spacer = "NNNNNNNNNN"
    assert m["sequence"] == [P.sub(A, 5)[:60] + spacer + A[40:], A[:60] + spacer + A[40:], A[:60] + spacer + P.sub(A, 50)[40:]]
    assert m["prefer"].tolist() == [NA] * 3 and m["nmatch"].tolist() == [0] * 3 and m["accept"].all()
    assert list(m)[9:] == ["F.n0", "R.n0", "F.birth_ham", "R.birth_ham"]
    assert [int(x) for x in m["F.n0"]] == [1, 5, 5] and [int(x) for x in m["R.n0"]] == [2, 2, 9]


def test_sample_without_pairs():
    m = R.merge_sample(*P.empty_sample())
    assert list(m) == list(R.merge_sample(*P.hand_sample()).keys()) and all(len(v) == 0 for v in m.values())


def test_non_corresponding_objects():
    dF, rF, dR, rR = P.hand_sample()
    bad = [(dF, P.derep_obj(4, rF["map"][:-1]), dR, rR),                       # lengths of mapF and mapR differ
           (P.dada_obj(["ACGT"], [1], [1, 1, 1]), rF, dR, rR),               # max(mapF) != length(dadaF$map)
           (dF, rF, dR, P.derep_obj(3, [1] * 9))]                            # max(mapR) != length(dadaR$map)
    for c in bad:
        with pytest.raises(ValueError, match="Non-corresponding derep-class and dada-class objects."):
            R.merge_sample(*c)


def test_mergepairs_argument_errors():
    from dada2_b200 import mergePairs
    dF, rF, dR, rR = P.hand_sample()
    with pytest.raises(ValueError, match="dadaF and dadaR must be provided as dada-class objects"):
        mergePairs(rF, rF, dR, rR)
    with pytest.raises(ValueError, match="derepF and derepR must be provided as derep-class objects"):
        mergePairs(dF, 3, dR, rR)
    with pytest.raises(ValueError, match="The dadaF/derepF/dadaR/derepR arguments must be the same length."):
        mergePairs([dF, dF], [rF, rF], [dR], [rR, rR])
    with pytest.raises(TypeError, match='formal argument "band" matched by multiple actual arguments'):
        mergePairs(dF, rF, dR, rR, band=16)
    with pytest.raises(ValueError, match="vec = TRUE"):
        mergePairs(dF, rF, dR, rR, vec=True)
    with pytest.raises(ValueError, match="endsfree = FALSE"):
        mergePairs(dF, rF, dR, rR, endsfree=False)
    with pytest.raises(TypeError, match="unused argument"):
        mergePairs(dF, rF, dR, rR, foo=1)
    with pytest.raises(ValueError, match="Incorrect format of \\$map"):
        mergePairs(dF, {"uniques": rF["uniques"], "map": rF["map"].astype(float)}, dR, rR)


def test_make_sequence_table_accepts_mergers(capsys):
    from dada2_b200.seqtab import makeSequenceTable
    m1 = {"sequence": ["CC", "AA", ""], "abundance": np.array([5, 3, 2]), "accept": np.array([True, True, False])}
    mat, cols, rows = makeSequenceTable(m1)
    assert cols == ["CC", "AA", ""] and mat.tolist() == [[5, 3, 2]] and rows is None
    assert capsys.readouterr().err == ""
    m2 = {"sequence": ["GG", "", "AA", ""], "abundance": np.array([4, 1, 7, 1])}
    mat, cols, rows = makeSequenceTable({"s1": m1, "s2": m2}, orderBy=None)
    assert "Duplicate sequences detected and merged." in capsys.readouterr().err
    assert cols == ["CC", "AA", "", "GG"] and rows == ["s1", "s2"]
    assert mat.tolist() == [[5, 3, 2, 0], [0, 7, 2, 4]]                     # tapply: "" + AA + GG, summed

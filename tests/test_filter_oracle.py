"""tests/filter_ref.py's C_matchRef and C_matrixEE pinned to the reference's src/filter.cpp, compiled unmodified into
oracle/_ref/libdada2ref_filter.so (oracle/filter.mk): hit counts exactly, EE bit for bit, on every generated read, at
word sizes 1 / 8 / 15 / 16 and both non_overlapping values.  Skipped where the reference library is not built."""
import numpy as np
import pytest

from tests import filter_cases as G
from tests import filter_ref as R

pytestmark = pytest.mark.skipif(R.ref_lib() is None, reason="oracle/_ref/libdada2ref_filter.so is not built")


def _reads():
    reads, _ = G.single_pool()
    syn = G.synthetic_reads(400, 250, seed=9)
    return reads + [G.read_at(syn, i) for i in range(len(syn) - 1)]


@pytest.mark.parametrize("w", [1, 8, 15, 16])
@pytest.mark.parametrize("nov", [True, False])
def test_match_ref_matches_reference(w, nov):
    seqs = [s for s, _ in _reads()]
    ph = G.phix()
    for ref in (ph, R.rc(ph)):
        assert np.array_equal(R.match_ref(seqs, ref, w, nov), R.ref_match_ref(seqs, ref, w, nov))


def test_matrix_ee_matches_reference_bit_for_bit():
    quals = [q for _, q in _reads()]
    got = [R.matrix_ee(q).hex() for q in quals]
    assert got == [x.hex() for x in R.ref_matrix_ee(quals)]
    assert any(R.matrix_ee(q) != R.tree_ee(q) for q in quals)       # a reordered sum would be caught


def test_golden_pool_values_are_the_references():
    g = G.load_golden()
    reads, _ = G.single_pool()
    assert [x.hex() for x in g["pool/ref_ee"]] == [R.matrix_ee(q).hex() for _, q in reads]
    assert np.array_equal(g["pool/ref_hits16"], R.match_ref([s for s, _ in reads], G.phix(), 16, True))

"""isShiftDenovo's restated R loop (tests/shift_ref.py) and the numpy restatement of the library's overlap filter in its
isShiftDenovo form, against the goldens made from the reference's own aligner -- CPU suite."""
import numpy as np
import pytest

from tests import shift_cases as K
from tests import shift_ref as S


def _golden_counts(seqs, g, name):
    where = {(seqs[i], seqs[j]): k for k, (i, j) in enumerate(zip(g[name + "_pq"], g[name + "_pp"]))}
    want = g[name + "_counts"]
    return lambda a, b: tuple(int(v) for v in want[where[(a, b)]])


@pytest.mark.parametrize("name", list(K.cases()))
def test_restated_loop_matches_goldens(name):
    g = K.load()
    seqs, ab = K.case(g, name)
    assert dict(zip(seqs, (int(a) for a in ab))) == K.cases()[name]
    for m in K.MIN_OVERLAPS:
        f = S.is_shift_denovo(dict(zip(seqs, (int(a) for a in ab))), minOverlap=m, counts=_golden_counts(seqs, g, name))
        assert np.array_equal([f[s] for s in seqs], g[K.flag_key(name, m)]), m
        # flagSubseqs is never passed on (R/chimeras.R:391)
        f2 = S.is_shift_denovo(dict(zip(seqs, (int(a) for a in ab))), minOverlap=m, flagSubseqs=True, counts=_golden_counts(seqs, g, name))
        assert f2 == f


def test_restated_loop_over_the_compiled_aligner():
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref not built")
    g = K.load()
    seqs, ab = K.case(g, "synthetic")
    f = S.is_shift_denovo(dict(zip(seqs, (int(a) for a in ab))), minOverlap=20)
    assert np.array_equal([f[s] for s in seqs], g[K.flag_key("synthetic", 20)])


def test_filter_never_rejects_a_shift_and_rejects_most_pairs():
    g = K.load()
    seqs, _ = K.case(g, "synthetic")
    q, p, c = g["synthetic_pq"], g["synthetic_pp"], g["synthetic_counts"]
    for m in K.MIN_OVERLAPS:
        flt = np.array([S.shift_filter(seqs[i], seqs[j], m) for i, j in zip(q, p)], bool)
        sh = np.array([S.is_shifted_pair(seqs[i], seqs[j], m, counts=lambda a, b, k=k: tuple(c[k])) for k, (i, j) in enumerate(zip(q, p))])
        assert not np.any(sh & ~flt), m
        if m == 20:
            assert np.count_nonzero(~flt) > 0.8 * len(q), (np.count_nonzero(~flt), len(q))

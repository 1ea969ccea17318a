"""collapseNoMismatch's restated R loop (tests/collapse_ref.py) and the numpy restatement of the library's screen and
overlap filter, against the goldens made from the reference's own nwhamming -- CPU suite."""
import numpy as np
import pytest

from tests import collapse_cases as G
from tests import collapse_ref as R


def _golden_nwhamming(name):
    seqs, pq, pr = G.pairs(name)
    pos = {s: k for k, s in enumerate(seqs)}
    tabs = {a: G.ham(name, *a) for a in G.aligners(name)}
    where = {(int(j), int(i)): x for x, (j, i) in enumerate(zip(pq, pr))}

    def nwhamming(s1, s2, vec=True, band=-1, **kw):
        return int(tabs[(int(vec), band)][where[(pos[s1], pos[s2])]])
    return nwhamming


@pytest.mark.parametrize("k", [k for k, _, _ in G.cases()])
def test_restated_loop_matches_goldens(k):
    _, name, o = G.cases()[k]
    mat, cols, _ = G.table(name)
    m, c = R.collapse(mat, cols, nwhamming=_golden_nwhamming(name), **o)
    wm, wc = G.expected(k)
    assert c == wc and np.array_equal(m, wm)


def test_restated_loop_with_port_nwhamming():
    for k, name, o in G.cases():
        mat, cols, _ = G.table(name)
        m, c = R.collapse(mat, cols, nwhamming=R.port_nwhamming, **o)
        wm, wc = G.expected(k)
        assert c == wc and np.array_equal(m, wm), (k, o)


@pytest.mark.parametrize("name", ["families", "repeats"])
def test_screen_and_filter_restatement_on_every_pair(name):
    seqs, pq, pr = G.pairs(name)
    for m in G.overlaps(name):
        got = np.array([R.screen(seqs[j], seqs[i], m) for j, i in zip(pq, pr)], np.int32)
        assert np.array_equal(got, G.scr(name, m))
    for v, b in G.aligners(name):
        h = G.ham(name, v, b)
        ver = np.array([R.overlap_filter(seqs[j], seqs[i], band=b) for j, i in zip(pq, pr)])
        assert not np.any(~ver & (h == 0)), "the filter rejected a pair with nwhamming 0"
        if b < 0:
            assert np.count_nonzero(~ver) > len(pq) // 2       # it does reject most unrelated and near pairs
        port = np.array([R.port_nwhamming(seqs[j], seqs[i], vec=bool(v), band=b) for j, i in zip(pq, pr)])
        assert np.array_equal(port, h), (name, v, b)


def test_greedy_resolution_matches_loop():
    """Resolving the loop from the ham-0 pairs alone gives the loop's representatives."""
    for name in ("families", "repeats"):
        seqs, pq, pr = G.pairs(name)
        for v, b in G.aligners(name):
            h = G.ham(name, v, b)
            scr = G.scr(name, 20) if 20 in G.overlaps(name) else G.scr(name, G.overlaps(name)[0])
            m = 20 if 20 in G.overlaps(name) else G.overlaps(name)[0]
            zero = [(int(j), int(i)) for j, i, s, x in zip(pq, pr, scr, h) if s and x == 0]
            rep = R.greedy(len(seqs), zero)
            kept = []
            want = []
            for j, q in enumerate(seqs):
                hit = next((i for i in kept if R.screen(q, seqs[i], m) and h[_idx(pq, pr, j, i)] == 0), None)
                want.append(j if hit is None else hit)
                if hit is None:
                    kept.append(j)
            assert rep.tolist() == want


def _idx(pq, pr, j, i):
    return int(np.nonzero((pq == j) & (pr == i))[0][0])


def test_eval_pair_equals_ham_on_reference_alignments():
    """For vec=TRUE the goldens take mismatch + indel from get_ham_endsfree; C_eval_pair agrees on the same alignments."""
    from oracle import ref
    if not ref.available():
        pytest.skip("the reference library is not built")
    seqs, pq, pr = G.pairs("repeats")
    for j, i in list(zip(pq, pr))[::3]:
        a0, a1 = ref.align(seqs[j], seqs[i], band=-1, mode=0)
        _, x, d = R.eval_pair(a0, a1)
        assert x + d == R.ref_nwhamming(seqs[j], seqs[i], vec=True, band=-1)

"""removePrimers' restatement (tests/primer_ref.py) against itself and the golden file -- CPU suite: the vectorised
matcher equals the per-shift definition on seeded random cases (IUPAC letters on both sides, k >= P, reads shorter
than the primer), and tests/golden/primer.npz equals the restatement on every case."""
import numpy as np

from tests import primer_cases as G
from tests import primer_ref as R


def test_vectorised_matcher_equals_the_literal_definition():
    rng = np.random.default_rng(42)
    letters = np.array(list(R.IUPAC))
    for t in range(4000):
        P = int(rng.integers(1, 12))
        iupac_p = rng.random() < 0.5
        p = "".join(rng.choice(letters if iupac_p else letters[:4], P))
        s = "".join(rng.choice(letters if rng.random() < 0.5 else letters[:4], int(rng.integers(0, 30))))
        if rng.random() < 0.3 and len(s) > P:                        # plant the primer with a few edits
            j = int(rng.integers(-2, len(s) - P + 3))
            planted = G.mutate(p, rng.choice(P, min(P, int(rng.integers(0, 3))), replace=False), rng) if "N" not in p else p
            s = (s[:max(j, 0)] + planted[max(-j, 0):] + s[j + P:])[:len(s) + 2]
        k = int(rng.integers(0, P + 3))
        assert R.match_vec(p, s, k) == R.match_literal(p, s, k), (p, s, k)


def test_rules_at_their_edges():
    assert R.min_shift(20, 2) == -2 and R.min_shift(3, 3) == -2 and R.min_shift(3, 5) == -2 and R.min_shift(4, 3) == -3
    assert R.match_literal("ACGT", "CGTTTT", 1) == [(0, 3)]                  # off the left end by 1 at k = 1
    assert R.match_literal("ACGT", "CGTTTT", 0) == []                        # k = 0: only placements inside the read
    assert R.match_literal("ACGT", "TTTACG", 1) == [(4, 7)]                  # off the right end
    assert R.match_literal("ACGT", "TTACGN", 0) == []                        # fixed: N in the read is a mismatch
    assert R.match_literal("ACGN", "TTACGN", 0) == [(3, 6)]                  # IUPAC primer: N matches
    assert R.match_literal("ACGR", "TTACGA", 0) == [(3, 6)] and R.match_literal("ACGR", "TTACGY", 0) == []
    assert R.match_literal("AC", "", 2) == [(0, 1)] and R.match_literal("AC", "", 1) == []   # k >= P: every placement, even on an empty read
    assert R.match_literal("ACG", "T", 5) == [(-1, 1), (0, 2), (1, 3)]


def test_golden_equals_the_restatement():
    g = G.load_golden()
    for case in G.cases():
        w = G.want_from_restatement(case)
        gw = G.want_from_golden(g, case)
        assert np.array_equal(gw["reason"], w["reason"]) and np.array_equal(gw["flags"], w["flags"]), case["name"]
        assert gw["skipped"] == w["skipped"] and gw["multi"] == w["multi"] and np.array_equal(gw["src"], w["src"]), case["name"]
        assert gw["seqs"] == w["seqs"] and [list(map(int, q)) for q in gw["quals"]] == w["quals"], case["name"]
        assert np.array_equal(g[case["name"] + "/hits"], G.restate_hits(case)), case["name"]


def test_vector_decide_equals_the_per_read_rules():
    for case in G.cases():
        w = G.restate(case)
        if w["skipped"]:
            continue
        h = G.restate_hits(case)
        rec = np.zeros(h.shape[:2], np.dtype([(f, np.int32) for f in ("count", "first_start", "first_end", "last_start", "last_end")]))
        for j, f in enumerate(rec.dtype.names):
            rec[f] = h[:, :, j]
        lens = [len(s) for s, _ in case["reads"]]
        reason, flags = R.vector_decide(rec, lens, case["pr"] is not None, case["trim_fwd"], case["trim_rev"], case["orient"])
        assert np.array_equal(reason, w["reason"]) and np.array_equal(flags, w["flags"]), case["name"]

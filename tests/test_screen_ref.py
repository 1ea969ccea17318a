"""Pins tests/screen_ref.py, the plain restatement of the k-mer screen that the screen stage tests compare the kernels with: on
every generated pair of tests/screen_cases.py up to 1500 nt, its decision must equal raw_align's in the CPU oracle
(oracle/port.cpp through oracle.port.pair) and, where oracle/_ref/libdada2ref.so is built, the reference's own kdist, kodist
and shroud decision."""
import numpy as np
import pytest

from oracle import port, ref
from tests import cases, screen_cases, screen_ref

PIN_MAXLEN = 1500              # oracle.port.pair keeps the full DP matrices: the 9998-nt pairs stay out


def _distinct_calls(case):
    seen = {}
    for call in case["calls"]:
        key = (call["centre"], call["kdist_cutoff"], tuple(sorted(call["opts"].items())))
        seen.setdefault(key, call)
    return list(seen.values())


@pytest.mark.parametrize("make", [screen_cases.boundary_case, screen_cases.bound_case, screen_cases.repeat_case, screen_cases.length_case],
                         ids=lambda f: f.__name__)
def test_screen_ref_matches_oracle_raw_align(make):
    case = make()
    seqs = case["seqs"]
    err = cases.tperr1()
    use_ref = ref.available()
    n = 0
    for call in _distinct_calls(case):
        o = dict(call["opts"])
        c = call["centre"]
        want = screen_ref.screen(seqs, c, call["kdist_cutoff"], **o)
        oo = dict(o)
        use_kmers = oo.pop("use_kmers", True)
        for r in range(len(seqs)):
            if max(len(seqs[c]), len(seqs[r])) > PIN_MAXLEN:
                continue
            p = port.pair(seqs[c], None, seqs[r], None, err, use_kmers=use_kmers, kdist_cutoff=call["kdist_cutoff"], homo_gap=-8, **oo)
            assert p["kind"] == want["kind"][r], (case["label"], c, r, call["kdist_cutoff"], o, p["kind"], want["kind"][r])
            if use_ref and use_kmers and r % 7 == 0:
                q = ref.pair(seqs[c], None, seqs[r], None, err, use_kmers=True, kdist_cutoff=call["kdist_cutoff"], **oo)
                assert q["shrouded"] == (want["kind"][r] == 0), (case["label"], c, r)
                assert q["kdist"] == want["kdist"][r], (case["label"], c, r, q["kdist"], want["kdist"][r])
                if oo.get("gapless", True) and oo.get("SSE", 2) != 0:         # the library reports kord_dist_SSEi's value
                    assert q["kodist"] == want["kodist"][r], (case["label"], c, r, q["kodist"], want["kodist"][r])
            n += 1
    assert n > 100


def test_screen_cases_reach_the_edges():
    """The generated cases contain what their names promise (so that a kernel bug there cannot pass unexercised)."""
    b = screen_cases.bound_case()
    w = screen_ref.screen(b["seqs"], 0, 0.42)
    lb = screen_ref.kdist_of(w["bound"], 120, np.array([len(s) for s in b["seqs"]]))
    inconclusive = ~(lb > 0.42)
    assert (inconclusive & w["shrouded"]).sum() > 200 and (inconclusive & ~w["shrouded"]).sum() > 200
    r = screen_cases.repeat_case()
    counts = [int(screen_ref.kmer_counts(s).max()) for s in r["seqs"]]
    for want in (2, 63, 64, 65, 260):
        assert want in counts, want
    nrep = [int((screen_ref.kmer_counts(s) >= 2).sum()) for s in r["seqs"]]
    for d in (0, 1, 7, 8, 9, 15, 16, 47, 48, 49):
        assert d in nrep, d
    ov = screen_ref.screen(r["seqs"], 0, 0.42)["overflow"]
    assert ov.any() and not ov.all()
    lens = {len(s) for s in screen_cases.length_case()["seqs"]}
    assert {6, 19, 20, 21, 250, 251, 1500} <= lens
    assert max(len(s) for s in screen_cases.long_case()["seqs"]) == screen_cases.MAXLEN

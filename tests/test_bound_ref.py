"""CPU checks of tests/bound_ref.py (the plain restatement of the two-phase loop NW's bound) and of the cases in tests/bound_cases.py:
the bound holds exactly on every generated pair, the vectorised raw factors equal a direct loop, and every case reaches the edges
its name promises."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import port
from tests import bound_cases as BC
from tests import bound_ref as BR

pytestmark = pytest.mark.skipif(not port.available(), reason="oracle/_ref/liboracle_port.so is not built")


@pytest.fixture(scope="module")
def emu_cases():
    cs = BC.all_cases("emu")
    for c in cs:
        for m in ("nw", "gl"):
            BC.prepare(c, m)
    return cs


def test_lambda_never_exceeds_the_exact_bound(emu_cases):
    n = 0
    for c in emu_cases:
        for m in ("nw", "gl"):
            p = BC.prepare(c, m)
            for lam, B in zip(p["lam"], p["B"]):
                if B is None or B is math.inf:
                    continue
                assert Fraction(float(lam)) * p["T"] <= B * (1 + Fraction(1, 10 ** 12)), (c["label"], m, lam, float(B))
                n += 1
    assert n > 2000


def test_raw_factors_match_a_direct_loop(emu_cases):
    for c in emu_cases:
        uq = c["opts"].get("use_quals", True)
        S, rho = BR.raw_factors(c["seqs"], c["quals"], c["err"], uq)
        qi = BR.round_quals(c["quals"])
        for r in range(0, len(c["seqs"]), 7):
            s, rh = BR.raw_factors_loop(c["seqs"][r], qi[r], c["err"], uq)
            assert (s == S[r] or (math.isnan(s) and math.isnan(S[r]))) and rh == rho[r], (c["label"], r, s, S[r], rh, rho[r])


def test_round_quals_follows_the_upload():
    q = np.array([[0.49999999999999994, 0.5, 1.5, np.nextafter(2.5, 0), 2.5, 39.5, np.nan]])
    assert BR.round_quals(q).tolist() == [[0, 1, 2, 2, 3, 40, 0]]


def test_decision_thresholds():
    B = Fraction(1, 1000)
    edge = B * BR.MARGIN * (1 + Fraction(1, 10 ** 11))
    e_up = float(edge)
    if Fraction(e_up) < edge:
        e_up = float(np.nextafter(e_up, math.inf))
    assert BR.decision(3, 1e-4, e_up, 1, B) == BR.DROP
    assert BR.decision(3, 1e-4, float(np.nextafter(float(edge), 0.0)), 1, B) in (BR.EITHER, BR.DROP)
    assert BR.decision(3, 1e-4, float(B), 1, B) == BR.EITHER
    assert BR.decision(3, 1e-3, float(np.nextafter(1e-3, 0.0)), 1, B) == BR.KEEP          # the reference stores it
    assert BR.decision(3, 0.0, math.inf, 1, Fraction(1, 10 ** 290)) == BR.KEEP             # below 1e-280
    assert BR.decision(3, 0.0, math.inf, 1, None) == BR.KEEP                                # 0 * inf
    assert BR.decision(3, 0.0, math.inf, 1, B, S_fp=0.0) == BR.KEEP
    assert BR.decision(3, 0.0, e_up, 1, B, S_fp=1e-310) == BR.EITHER                        # subnormal S_r: 1e-6 of slack
    assert BR.decision(3, 0.0, float(B * 2), 1, B, S_fp=1e-310) == BR.DROP


def test_bound_cases_reach_the_edges(emu_cases):
    """Each case reaches what it promises: keep / drop / either jobs, underflowing and undefined bounds, identical pairs, subnormal
    S_r, warps whose ballot mixes kept and dropped jobs, hand-backs; and the GPU set has a list longer than k_nwlane takes."""
    for c in emu_cases:
        e = BC.edge_counts(c, "nw")
        for what in c["promises"]:
            assert e[what] > 0, (c["label"], what, e)
        assert e["either"] <= 0.3 * len(c["jobs"]), (c["label"], e)
    big = [c for c in BC.illumina_cases("gpu") if "over16k" in c["promises"]]
    assert len(big) == 1 and len(big[0]["jobs"]) > BC.LANE_MAX


def test_oracle_pairs_match_the_reference_on_a_sample(emu_cases):
    """ns and lambda come from oracle.port.pair; where the reference's own library is built, spot-check them against it."""
    from oracle import ref
    if not ref.available():
        pytest.skip("the reference's library is not built")
    n = 0
    for c in emu_cases[:3]:
        qi = BR.round_quals(c["quals"])
        cen = c["centre"]
        p = BC.prepare(c, "nw")
        for k in range(0, len(c["jobs"]), 11):
            r = int(c["jobs"][k])
            got = ref.pair(c["seqs"][cen], qi[cen, :len(c["seqs"][cen])].astype(np.uint8), c["seqs"][r], qi[r, :len(c["seqs"][r])].astype(np.uint8),
                           c["err"], use_kmers=False, band_size=c["opts"].get("band_size", 16))
            assert got["nsubs"] == p["ns"][k] and got["lam"] == p["lam"][k], (c["label"], r)
            n += 1
    assert n > 20

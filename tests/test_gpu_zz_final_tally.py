"""The final pass's diagonal-list tally (dd_final.cu) and round 0 through the two-phase diagonal test on the H100: the samples of
tests/final_tally_cases.py (also at several DADA2B_LANE_MAX settings), and a 1e5-unique run of the bench generator whose full output
is compared with the reference's own C++ (oracle/_ref) when it has been built."""
import os

import numpy as np
import pytest

from tests import cases
from tests import final_tally_cases as F

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", F.NAMES)
def test_final_tally_matches_reference(name):
    import dada2_b200
    F.run_case(name, dada2_b200.dada_uniques)


@pytest.mark.parametrize("lane_max", ["0", "32"])
@pytest.mark.parametrize("name", ["big_cluster", "indels_ragged"])
def test_round0_kernels_by_lane_max(monkeypatch, name, lane_max):
    import dada2_b200
    monkeypatch.setenv("DADA2B_LANE_MAX", lane_max)
    F.run_case(name, dada2_b200.dada_uniques)


def test_1e5_uniques_match_reference_cpp():
    from oracle import ref
    from tools import synth
    import dada2_b200
    if not ref.available():
        pytest.skip("oracle/_ref (the reference's own C++) is not built")
    seqs, ab, q, _ = synth.illumina(100000, seed=2024)
    err = cases.tperr1()
    got = dada2_b200.dada_uniques(seqs, ab, None, err, q)
    ref.set_threads(max(1, len(os.sched_getaffinity(0))))
    want = ref.dada_uniques(seqs, ab, None, err, q, multithread=True)
    for k in ("subqual", "map"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(want[k])), k
    for k in ("n0", "n1"):
        assert np.array_equal(got["clustering"][k], want["clustering"][k]), k
    a, b = np.asarray(got["clusterquals"]), np.asarray(want["clusterquals"])
    assert a.shape == b.shape and np.allclose(a, b, rtol=1e-10, atol=0, equal_nan=True)
    cases.assert_same(got, want, rtol=1e-10, label="1e5")

"""BASELINE-size checks on the GPU (configs[1]: 1e5 synthetic 250-nt uniques): size-independent properties
(tests/properties.py, pinned on the oracle at small sizes), run-to-run determinism, one-shot == resident, and the output
against the reference's own C++ on the same 1e5 uniques (tests/golden/e2e_fullsize_1e5.npz, tools/make_golden_fuzz.py:
every field, with map and pval at a seeded sample of raws).  bench.py diffs the 1e6 workload against the same library in its
cpu_baseline leg."""
import numpy as np
import pytest

from tests import cases
from tests.properties import check_invariants

pytestmark = pytest.mark.gpu


def workload():
    """-> (seqs, abundances, quals, err, truth)"""
    from tools import synth
    seqs, ab, q, truth = synth.illumina(100000, seed=12345)
    return seqs, ab, q, cases.tperr1(), truth


def sample_raws(n, k=20000):
    """The raws whose map / pval entries the golden keeps."""
    return np.sort(np.random.default_rng(5).choice(n, k, replace=False))


def test_1e5_uniques_invariants_determinism_and_paths_agree():
    import dada2_b200
    from tests.test_oracle import load_golden
    seqs, ab, q, err, truth = workload()
    res = dada2_b200.Resident(seqs, ab, None, q)
    a = res.run(err)
    b = res.run(err)
    res.close()
    c = dada2_b200.dada_uniques(seqs, ab, None, err, q)          # one-shot C-ABI path
    cases.assert_same(b, a, rtol=0.0, label="rerun")
    cases.assert_same(c, a, rtol=0.0, label="one-shot vs resident")
    check_invariants(seqs, ab, a)
    found = set(a["clustering"]["sequence"])
    assert len(found) == 100 and sum(v in found for v in truth["variants"]) >= 95     # the planted variants are recovered
    idx = sample_raws(len(seqs))
    got = dict(a, map=np.asarray(a["map"])[idx], pval=np.asarray(a["pval"])[idx])
    cases.assert_same(got, load_golden("fullsize_1e5"), rtol=1e-10, label="1e5 uniques vs the reference's C++")
    st = a["stats"]
    assert st["gpu_launches"] > 1000 and st["n_nw"] > 1_000_000 and st["n_final_nw"] == 100000
    cases.assert_same_screen_counts(a, oracle_counts(), label="1e5 uniques")


def oracle_counts():
    """The k-mer screen's totals on this workload from the CPU oracle (tools/make_golden_fuzz.py)."""
    import json
    import os
    return json.load(open(os.path.join(cases.GOLDEN, "e2e_fullsize_1e5_counts.json")))


def test_1e5_uniques_at_three_sms(monkeypatch):
    """DADA2B_SMS=3: the streaming screen runs 9 CTAs over 782 tiles (about 87 per CTA, the 4-stage ring wraps about 21 times) and
    every grid-stride kernel of the round takes many jobs per thread; output and screen counts stay the reference's."""
    import dada2_b200
    from tests.test_oracle import load_golden
    monkeypatch.setenv("DADA2B_SMS", "3")
    seqs, ab, q, err, truth = workload()
    res = dada2_b200.Resident(seqs, ab, None, q)
    a = res.run(err)
    res.close()
    idx = sample_raws(len(seqs))
    got = dict(a, map=np.asarray(a["map"])[idx], pval=np.asarray(a["pval"])[idx])
    cases.assert_same(got, load_golden("fullsize_1e5"), rtol=1e-10, label="1e5 uniques at 3 SMs")
    cases.assert_same_screen_counts(a, oracle_counts(), label="1e5 uniques at 3 SMs")

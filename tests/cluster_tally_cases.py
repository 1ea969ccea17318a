"""The per-cluster tallies of dada()'s output (dd_final.cu: k_cluster_tally) and repeated runs of one resident sample, shared by
tests/test_emu_cluster_tally.py (host SIMT emulator) and tests/test_gpu_zz_cluster_tally.py (H100).

The device counts abundance, n0, n1, nunq and the largest member abundance per cluster, and writes $map, from the final cluster of
every raw and its correct flag.  restated() recomputes abundance and nunq from the returned $map and the input abundances; n0 and
n1 (which need the final nsubs of every raw) are compared with the reference's result instead.
"""
import numpy as np

from tests import cases
from tests import final_tally_cases as F

GOLDEN_NAMES = ["syn800_omegaC", "syn800_singletons"]


def restated(result, ab):
    """abundance and nunq per cluster from $map (1-based cluster, INT_MIN where the raw is not correct)."""
    m = np.asarray(result["map"]).astype(np.int64)
    nclust = len(result["clustering"]["abundance"])
    ok = m >= 1
    assert np.all((m[ok] >= 1) & (m[ok] <= nclust))
    assert np.all(m[~ok] == np.iinfo(np.int32).min)
    ab = np.asarray(ab, dtype=np.int64)
    abundance = np.bincount(m[ok] - 1, weights=ab[ok], minlength=nclust).astype(np.int64)
    nunq = np.bincount(m[ok] - 1, minlength=nclust).astype(np.int64)
    return abundance, nunq


def check_tallies(result, ab):
    cl = result["clustering"]
    abundance, nunq = restated(result, ab)
    assert np.array_equal(np.asarray(cl["abundance"], dtype=np.int64), abundance)
    assert np.array_equal(np.asarray(cl["nunq"], dtype=np.int64), nunq)
    n0, n1 = np.asarray(cl["n0"], dtype=np.int64), np.asarray(cl["n1"], dtype=np.int64)
    assert np.all(n0 >= 0) and np.all(n1 >= 0) and np.all(n0 + n1 <= abundance)


def run_golden(name, dada_uniques):
    from tests.test_oracle import load_golden
    seqs, ab, pri, err, q, opts = cases.build_case(name)
    got = dada_uniques(seqs, ab, pri, err, q, **opts)
    want = load_golden(name)
    cases.assert_same(got, want, rtol=1e-10, label=name)
    check_tallies(got, ab)


def run_sample(name, dada_uniques):
    """final_tally_cases' samples: more clusters than are counted in shared memory, and raws made not correct by omegaC."""
    seqs, ab, q, opts = F.sample(name)
    want = F.expected(seqs, ab, q, opts)
    F.check_shape(name, want)
    check_tallies(want, ab)                  # the restatement holds for the reference ...
    got = dada_uniques(seqs, ab, None, cases.tperr1(), q, **opts)
    cases.assert_same(got, want, rtol=1e-10, label=name)
    check_tallies(got, ab)                   # ... and for the device tallies


def assert_identical(got, want, label):
    """Every output field equal, fp64 bit for bit (NaN where NaN)."""
    g, w = cases.flatten(got), cases.flatten(want)
    assert sorted(g) == sorted(w), label
    for k in g:
        a, b = np.asarray(g[k]), np.asarray(w[k])
        assert a.shape == b.shape, "%s %s shape %s vs %s" % (label, k, a.shape, b.shape)
        if a.dtype == np.float64:
            assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), "%s %s differs" % (label, k)
        else:
            assert np.array_equal(a, b), "%s %s differs" % (label, k)


# (options, DADA2B_SYNC_REPLAY) of the consecutive runs on one resident sample
REPEAT_RUNS = [({}, False), (dict(max_clust=3), False), (dict(omegaC=1e-2, omegaA=1e-20), True), ({}, True), (dict(max_clust=2), False)]


def run_repeated(monkeypatch):
    """Consecutive runs of one Resident with different options; each equals the same run on a fresh context."""
    import dada2_b200
    seqs, ab, q, _ = F.sample("omegaC")
    err = cases.tperr1()
    res = dada2_b200.Resident(seqs, ab, None, q)
    try:
        for k, (opts, sync_replay) in enumerate(REPEAT_RUNS):
            if sync_replay:
                monkeypatch.setenv("DADA2B_SYNC_REPLAY", "1")
            else:
                monkeypatch.delenv("DADA2B_SYNC_REPLAY", raising=False)
            got = res.run(err, **opts)
            fresh = dada2_b200.Resident(seqs, ab, None, q)
            try:
                want = fresh.run(err, **opts)
            finally:
                fresh.close()
            assert_identical(got, want, "run %d %s" % (k, opts))
            check_tallies(got, ab)
    finally:
        res.close()

"""GPU parity tests (run on an H100: pytest -m gpu).  Everything goes through the C-ABI of
libdada2b.so (include/dada2b.h, include/dada2b_test.h); the checker is the CPU oracle
(oracle/port.cpp) and the committed reference goldens (tests/golden)."""
import json
import os

import numpy as np
import pytest

from tests import cases
from tests.test_oracle import load_golden, _pairs

pytestmark = pytest.mark.gpu


def _api():
    import dada2_b200
    return dada2_b200


def ops_to_strings(ops, nops, a, b):
    al0, al1, i, j = [], [], 0, 0
    for c in ops[:nops]:
        if c == 1:
            al0.append(a[i]); al1.append(b[j]); i += 1; j += 1
        elif c == 2:
            al0.append("-"); al1.append(b[j]); j += 1
        elif c == 3:
            al0.append(a[i]); al1.append("-"); i += 1
        else:
            raise AssertionError("bad op %d" % c)
    assert i == len(a) and j == len(b)
    return "".join(al0), "".join(al1)


def test_device_calc_pA_matches_oracle():
    """ppois/calc_pA device function vs the oracle's R-nmath restatement: <= 1e-10 relative (contract),
    exact zeros agree."""
    from oracle import port
    api = _api()
    rng = np.random.default_rng(3)
    reads, E, prior = [], [], []
    for r in (1, 2, 3, 5, 10, 17, 50, 137, 1000, 20000, 300000):
        for e in (1e-300, 1e-30, 1e-8, 1e-3, 0.5, 1.0, 3, 50, 137, 999, 1001, 1e5, 1e7):
            for p in (0, 1):
                reads.append(r); E.append(e); prior.append(p)
    for _ in range(20000):
        r = int(10 ** rng.uniform(0, 5.7))
        e = r * 10 ** rng.uniform(-6, 0.5) if rng.random() < 0.7 else 10 ** rng.uniform(-20, 7)
        reads.append(r); E.append(float(e)); prior.append(int(rng.random() < 0.5))
    got = api.api.test_calc_pA(reads, E, prior)
    L = port.lib()
    want = np.array([L.port_calc_pA(r, e, p) for r, e, p in zip(reads, E, prior)])
    assert np.array_equal(got == 0, want == 0)
    nz = want != 0
    rel = np.abs(got[nz] - want[nz]) / np.abs(want[nz])
    assert rel.max() <= 1e-10, rel.max()


def test_pair_corpus_kernels_match_reference():
    """k_classify + k_align on the pair corpus: shroud/gapless/NW decision, alignment strings,
    nsubs and substitutions bit-exact; lambda bit-exact (same sequential fp64 product)."""
    api = _api()
    z, modes, a, b, qa, qb = _pairs()
    err = cases.tperr1()
    n = len(a)
    seqs = a + b
    maxlen = max(len(s) for s in seqs)
    q = np.full((2 * n, maxlen), np.nan)
    for i in range(n):
        q[i, :len(a[i])] = qa[i]
        q[n + i, :len(b[i])] = qb[i]
    res = api.Resident(seqs, np.ones(2 * n, np.int32), None, q)
    centre = np.arange(n, dtype=np.uint32)
    raw = centre + n
    nw = 0
    for m, o in modes.items():
        o = dict(o)
        r = res.test_pairs(centre, raw, err, use_kmers=True, kdist_cutoff=0.42, maxlen=maxlen, **o)
        for i in range(n):
            want_al0, want_al1 = str(z[m + "__al0"][i]), str(z[m + "__al1"][i])
            want_ns = int(z[m + "__nsubs"][i])
            if want_ns < 0:
                assert r["kind"][i] == 0, (m, i)
                continue
            assert r["kind"][i] in (1, 2), (m, i)
            al0, al1 = ops_to_strings(r["ops"][i], r["nops"][i], a[i], b[i])
            assert (al0, al1) == (want_al0, want_al1), (m, i, al0, want_al0, al1, want_al1)
            assert r["nsubs"][i] == want_ns, (m, i)
            assert r["lam"][i] == float(z[m + "__lam"][i]), (m, i, r["lam"][i], float(z[m + "__lam"][i]))
            nw += r["kind"][i] == 2
    assert nw > 200
    res.close()


def test_pair_corpus_loop_aligners_match_traceback_kernel():
    """The kernels that dominate device time never produce an alignment string, so they get their own stage test: every pair
    of the corpus, alone, through k_nwrow<EXACT>, k_nwlane, k_nwfwd and k_nwrow<BOUND> (dada2b_test_loop_nw) must give the
    (lambda, nsubs) of the warp-per-pair traceback kernel -- which the test above pins to the reference's alignments -- bit for
    bit, in every option set of the corpus (bands 8 / 16 / 32 / > len, score sets, homopolymer gap costs, unequal lengths)."""
    api = _api()
    z, modes, a, b, qa, qb = _pairs()
    err = cases.tperr1()
    n = len(a)
    seqs = a + b
    maxlen = max(len(s) for s in seqs)
    q = np.full((2 * n, maxlen), np.nan)
    for i in range(n):
        q[i, :len(a[i])] = qa[i]
        q[n + i, :len(b[i])] = qb[i]
    res = api.Resident(seqs, np.ones(2 * n, np.int32), None, q)
    centre = np.arange(n, dtype=np.uint32)
    raw = centre + n
    took = {0: 0, 1: 0, 2: 0, 3: 0}
    more = {"vec8": {"band_size": 8}, "vec32": {"band_size": 32}, "sc8_scores": {"band_size": 8, "match": 4, "mismatch": -5, "gap": -7}}
    for m, o in list(modes.items()) + list(more.items()):
        o = dict(o)
        if o.get("band_size", 16) < 0:
            continue                                             # unbanded: k_align only
        want = res.test_pairs(centre, raw, err, use_kmers=False, kdist_cutoff=0.42, maxlen=maxlen, **o)
        assert np.all(want["kind"] == (1 if o.get("band_size", 16) == 0 else 2)), m
        if o.get("band_size", 16) == 0:
            continue
        for which in (0, 1, 2, 3):
            r = res.test_loop_nw(which, centre, raw, err, **o)
            for i in range(n):
                if not r["handled"][i]:
                    continue
                took[which] += 1
                assert r["nsubs"][i] == want["nsubs"][i], (m, which, i, r["nsubs"][i], want["nsubs"][i])
                if which != 3:
                    assert r["lam"][i] == want["lam"][i], (m, which, i, r["lam"][i], want["lam"][i])
            if which in (0, 1, 3):                               # the row / lane kernels take exactly the equal-length pairs of their bands
                homo = o.get("vectorized_alignment", True) is False and o.get("homo_gap", o.get("gap", -8)) != o.get("gap", -8)
                ok_band = o.get("band_size", 16) in (8, 16, 32) and not homo
                for i in range(n):
                    fits = ok_band and len(a[i]) == len(b[i]) and len(a[i]) >= o.get("band_size", 16) + 2
                    assert bool(r["handled"][i]) == fits, (m, which, i, len(a[i]), len(b[i]))
    assert took[0] > 100 and took[1] > 100 and took[2] > 200 and took[3] > 100, took
    res.close()


def test_config1_bit_identical():
    api = _api()
    seqs, ab, q = cases.load_config1()
    got = api.dada_uniques(seqs, ab, None, cases.tperr1(), q)
    want = load_golden("config1")
    cases.assert_same(got, want, rtol=1e-10, label="config1")
    assert len(got["clustering"]["sequence"]) == 10
    assert (got["stats"]["n_align"], got["stats"]["n_shroud"]) == (8655, 3032)          # the oracle's counts (tests/test_oracle.py)


@pytest.mark.parametrize("name,tail_smem", [pytest.param(name, None, id=name) for name in sorted(cases.E2E_CASES)] +
                         [pytest.param(name, n, id=f"{name}-tail_smem{n}") for name in ("syn800_default", "syn700_ragged", "syn800_priors")
                          for n in ("0", "12")])
def test_e2e_matches_reference_golden(name, tail_smem):
    """tail_smem: DADA2B_TAIL_SMEM_CLUSTERS (test hook), the round tail's per-cluster state in global memory from the first round (0)
    or from mid-run (12), as runs past ~32 k clusters do."""
    api = _api()
    seqs, ab, pri, err, q, opts = cases.build_case(name)
    with pytest.MonkeyPatch.context() as mp:
        if tail_smem is not None:
            mp.setenv("DADA2B_TAIL_SMEM_CLUSTERS", tail_smem)
        got = api.dada_uniques(seqs, ab, pri, err, q, **opts)
    _check_e2e(name, got)


def _check_e2e(name, got):
    seqs, ab, pri, err, q, opts = cases.build_case(name)
    want = load_golden(name)
    pb = None
    if pri is not None:
        pb = np.zeros(len(want["clustering"]["sequence"]), dtype=bool)
        pb[1:] = want["clustering"]["birth_pval"][1:] >= opts.get("omegaA", 1e-40)
    cases.assert_same(got, want, rtol=1e-10, prior_born=pb, label=name)
    cases.assert_same_screen_counts(got, cases.oracle_screen_counts(name), label=name)


@pytest.mark.parametrize("sms", ["1", "2"])
@pytest.mark.parametrize("name", sorted(cases.E2E_CASES) + ["config1"])
def test_e2e_golden_at_capped_sm_count(monkeypatch, name, sms):
    """DADA2B_SMS (test hook, read at upload) caps the SM count every grid of dada() is sized from: golden-sized inputs then give each
    CTA many tiles / jobs (the streaming screen's ring wraps, grid-stride loops run several times), as the 1e6 workload does."""
    api = _api()
    monkeypatch.setenv("DADA2B_SMS", sms)
    if name == "config1":
        seqs, ab, q = cases.load_config1()
        res = api.Resident(seqs, ab, None, q)
        got = res.run(cases.tperr1())
        res.close()
        cases.assert_same(got, load_golden("config1"), rtol=1e-10, label="config1 at %s SMs" % sms)
        assert (got["stats"]["n_align"], got["stats"]["n_shroud"]) == (8655, 3032)
        return
    seqs, ab, pri, err, q, opts = cases.build_case(name)
    res = api.Resident(seqs, ab, pri, q)
    got = res.run(err, **opts)
    res.close()
    _check_e2e(name, got)


@pytest.mark.parametrize("blk", [1, 100])
def test_upload_pipeline_many_blocks(monkeypatch, blk):
    """do_upload pipelines packing (worker threads, blocks of raws) with grouped H2D copies from the pinned staging buffers:
    DADA2B_PACK_BLK (test hook) makes 800 raws span many blocks and copy groups; one-shot call and re-upload."""
    api = _api()
    monkeypatch.setenv("DADA2B_PACK_BLK", str(blk))
    for name in ("syn800_default", "syn700_ragged"):
        seqs, ab, pri, err, q, opts = cases.build_case(name)
        want = load_golden(name)
        cases.assert_same(api.dada_uniques(seqs, ab, pri, err, q, **opts), want, rtol=1e-10, label=name)
        from dada2_b200 import _abi
        r = api.Resident(seqs[::-1], ab[::-1].copy(), None, q[::-1].copy())
        r.reupload(_abi.PackedIn(seqs, ab, pri, None, q))
        cases.assert_same(r.run(err, **opts), want, rtol=1e-10, label=name + " after reupload")
        r.close()


def test_resident_rerun_is_deterministic_and_err_swappable():
    api = _api()
    seqs, ab, pri, err, q, opts = cases.build_case("syn800_default")
    r = api.Resident(seqs, ab, pri, q)
    a = r.run(err, **opts)
    b = r.run(err, **opts)
    cases.assert_same(a, b, rtol=0.0, label="rerun")
    ones = r.run(np.ones((16, 41)), max_clust=1)
    want = load_golden("syn800_ones_err")  # different seed: only structural check here
    assert len(ones["clustering"]["sequence"]) == 1
    r.close()


def test_error_paths():
    api = _api()
    with pytest.raises(api.Dada2bError, match="16 rows"):
        api.dada_uniques(["ACGTACGTAC"], [1], None, np.ones((15, 41)), np.full((1, 10), 30.0))
    with pytest.raises(api.Dada2bError, match="kmer-size"):
        api.dada_uniques(["ACGTA"], [1], None, np.ones((16, 41)), np.full((1, 5), 30.0))
    with pytest.raises(api.Dada2bError, match="Unexpected nucleotide"):
        api.dada_uniques(["ACGTNCGTAC"], [1], None, np.ones((16, 41)), np.full((1, 10), 30.0))
    with pytest.raises(api.Dada2bError, match="exceeded range"):
        api.dada_uniques(["ACGTACGTAC"], [1], None, np.ones((16, 41)), np.full((1, 10), 60.0))
    with pytest.raises(api.Dada2bError, match="Zero input"):
        api.dada_uniques([], [], None, np.ones((16, 41)), np.zeros((0, 10)))

"""Sample pooling (dd_pool.cu) and dada() / learnErrors() over samples (dada2_b200/denoise.py) on the H100: every pooling
case of tests/pool_cases.py plus 8 samples of 2.4e5 sample-uniques bit-identical to the host combineDereps2, the man
page's two-sample example pass by pass, pool = TRUE and pool = "pseudo" against dada_uniques run by hand, and learnErrors'
sample cut-off."""
import os

import numpy as np
import pytest

from tests import cases
from tests import pool_cases as P

pytestmark = pytest.mark.gpu
GOLDEN = cases.GOLDEN
FILES = [os.path.join(GOLDEN, f) for f in ("sam1F.fastq.gz", "sam2F.fastq.gz")]


def _sam():
    from dada2_b200 import derep
    return [derep.derepFastq(f) for f in FILES]


def big_dereps(nsamp=8, npool=60000, per=30000, L=250, seed=9):
    """nsamp samples drawing `per` uniques each from `npool` 250-nt sequences (some truncated to proper prefixes), with
    fractional means, random abundances and maps: the radix tiles and the segments cross block boundaries."""
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, 4, (npool, L)).astype(np.uint8)
    lut = np.frombuffer(b"ACGT", np.uint8)
    lens = np.where(rng.random(npool) < 0.2, L - rng.integers(1, 12, npool), L)
    seqs = [lut[codes[i, :lens[i]]].tobytes().decode() for i in range(npool)]
    for i in range(0, npool // 10, 2):                            # exact proper prefixes of other pooled sequences
        seqs[i + 1] = seqs[i][:L - 7]
    seqs = list(dict.fromkeys(seqs))
    out = []
    for s in range(nsamp):
        pick = rng.choice(len(seqs), per, replace=False)
        ml = int(max(len(seqs[i]) for i in pick))
        q = rng.integers(4, 80, (per, ml)) / 2.0
        q[np.arange(ml)[None, :] >= np.array([len(seqs[i]) for i in pick])[:, None]] = np.nan
        out.append({"uniques": [seqs[i] for i in pick], "abundances": rng.integers(1, 60, per).astype(np.int32), "quals": q,
                    "map": rng.integers(1, per + 1, 20000).astype(np.int32)})
    return out


def test_pool_kernels_match_combineDereps2():
    from dada2_b200.derep import pool_dereps
    P.check_all(big=True)
    P.check_refusals()
    ds = big_dereps()
    pr = P.random_priors(ds, 1)
    got = pool_dereps(ds, priors=pr, return_stats=True)
    assert sum(len(d["uniques"]) for d in ds) >= 200000
    P.assert_same(got, P.expected(ds, pr), "8 samples x 30000 uniques")
    st = got["stats"]
    print("pool 8 x 30000 -> %d: kernels %.2f ms, h2d %.2f ms (%d B), d2h %.2f ms (%d B)" % (
        len(got["uniques"]), st["ms_kernels"], st["ms_h2d"], st["h2d_bytes"], st["ms_d2h"], st["d2h_bytes"]))


def _by_hand_pass(ds, err):
    """One pass of dada()'s loop written out: per-sample dada_uniques with err extended to each sample's qmax."""
    import dada2_b200
    from dada2_b200.denoise import extend_err
    out = []
    for d in ds:
        qmax = int(np.ceil(np.nanmax(d["quals"])))
        out.append(dada2_b200.dada_uniques(d["uniques"], d["abundances"], None, extend_err(err, qmax), d["quals"]))
    return out


def test_man_page_example_pass_by_pass():
    import dada2_b200
    from dada2_b200.errmodel import accumulateTrans, loessErrfun
    from tests.test_oracle import load_golden
    d1, d2 = _sam()
    tperr1 = cases.tperr1()
    r = dada2_b200.dada({"sam1": d1, "sam2": d2}, err=tperr1, selfConsist=True)
    assert list(r) == ["sam1", "sam2"]
    errs = r["sam1"]["err_in"]
    assert np.array_equal(errs[0], tperr1) and r["sam1"]["passes"] == len(errs)
    for k, e in enumerate(errs):
        res = _by_hand_pass([d1, d2], e)
        est = loessErrfun(accumulateTrans([x["subqual"] for x in res]))
        nxt = errs[k + 1] if k + 1 < len(errs) else r["sam1"]["err_out"]
        assert np.array_equal(est, nxt), "pass %d refit" % k
    for name, want in zip(("sam1", "sam2"), res):
        cases.assert_same(r[name], want, rtol=0, label="last pass " + name)
        assert r[name]["denoised"] == dict(zip(want["clustering"]["sequence"], want["clustering"]["abundance"].tolist()))
    one = dada2_b200.dada([d1, d2], err=tperr1)
    cases.assert_same(one[0], load_golden("config1"), rtol=1e-10, label="selfConsist=False sam1 vs config-1 golden")
    assert np.array_equal(one[0]["err_in"], tperr1)


def _expand_by_hand(pooled_res, pooled_uniques, d):
    """R/dada.R:443-475 written with loops and dicts."""
    pos = {s: i for i, s in enumerate(pooled_uniques)}
    m = [int(pooled_res["map"][pos[s]]) for s in d["uniques"]]
    keep = sorted({v for v in m if v != P.NA_INT})
    newBi = {old: k + 1 for k, old in enumerate(keep)}
    den = {}
    for v, a in zip(m, d["abundances"]):
        if v != P.NA_INT:
            s = pooled_res["clustering"]["sequence"][v - 1]
            den[s] = den.get(s, 0) + int(a)
    bs = [(newBi[c], p) for c, p in zip(pooled_res["birth_subs"]["clust"], pooled_res["birth_subs"]["pos"]) if c in newBi]
    return {"denoised": den, "map": [newBi.get(v, P.NA_INT) for v in m], "birth_subs": bs,
            "sequence": [pooled_res["clustering"]["sequence"][c - 1] for c in keep]}


def test_pool_true_equals_dada_uniques_on_the_pooled_derep():
    import dada2_b200
    from dada2_b200.derep import combineDereps2
    from dada2_b200.denoise import extend_err
    d1, d2 = _sam()
    tperr1 = cases.tperr1()
    r = dada2_b200.dada([d1, d2], err=tperr1, pool=True)
    pooled = combineDereps2([d1, d2])
    want = dada2_b200.dada_uniques(pooled["uniques"], pooled["abundances"], None,
                                   extend_err(tperr1, int(np.ceil(np.nanmax(pooled["quals"])))), pooled["quals"])
    assert np.array_equal(r[0]["pval"], want["pval"]) and np.array_equal(r[0]["trans"], want["subqual"])
    tot = {}
    for d, got in zip((d1, d2), r):
        h = _expand_by_hand(want, pooled["uniques"], d)
        assert got["denoised"] == h["denoised"] and got["sequence"] == h["sequence"]
        assert got["map"].tolist() == h["map"]
        assert list(zip(got["birth_subs"]["clust"].tolist(), got["birth_subs"]["pos"].tolist())) == h["birth_subs"]
        for s, a in got["denoised"].items():
            tot[s] = tot.get(s, 0) + a
    if (want["map"] != P.NA_INT).all():                         # without NA maps every pooled read lands in some sample's cluster
        assert tot == dict(zip(want["clustering"]["sequence"], want["clustering"]["abundance"].tolist()))
    full = dada2_b200.dada([d1, d2], err=tperr1, pool=True, selfConsist=True)
    assert len(full[0]["err_in"]) >= 2


def _noqual(trans):
    """A quality-blind refit (rates aggregated over qualities, one pseudo-count), enough for data of one quality score."""
    obs = np.asarray(trans, np.float64).sum(axis=1) + 1.0
    rate = obs.reshape(4, 4) / obs.reshape(4, 4).sum(axis=1, keepdims=True)
    return np.repeat(rate.reshape(16, 1), np.asarray(trans).shape[1], axis=1)


def _pseudo_samples():
    """A, B, C and a one-substitution variant V of A: V is called in samples 1 and 2 on its own, and is present with
    3 reads in sample 3, too few to call there without a prior."""
    rng = np.random.default_rng(4)
    A = "".join("ACGT"[i] for i in rng.integers(0, 4, 120))
    V = A[:60] + {"A": "C", "C": "G", "G": "T", "T": "A"}[A[60]] + A[61:]
    B = "".join("ACGT"[i] for i in rng.integers(0, 4, 120))
    C = "".join("ACGT"[i] for i in rng.integers(0, 4, 120))
    def d(seqs, ab):
        return {"uniques": seqs, "abundances": np.array(ab, np.int32), "quals": np.full((len(seqs), 120), 38.0),
                "map": np.arange(1, len(seqs) + 1, dtype=np.int32)}
    return [d([A, B, V], [1000, 500, 200]), d([A, C, V], [900, 400, 150]), d([A, B, C, V], [800, 300, 200, 3])], V


def test_pool_pseudo_second_pass_with_pseudo_priors():
    import dada2_b200
    from dada2_b200.errmodel import accumulateTrans
    from dada2_b200.seqtab import makeSequenceTable
    ds, V = _pseudo_samples()
    err = np.full((16, 41), 1e-3); err[[0, 5, 10, 15]] = 1 - 3e-3
    p1 = _by_hand_pass(ds, err)
    assert V not in p1[2]["clustering"]["sequence"] and V in p1[0]["clustering"]["sequence"]
    mat, cols, _ = makeSequenceTable([{"clustering": x["clustering"]} for x in p1])
    rule = sorted(c for c, k in zip(cols, (mat > 0).sum(axis=0) >= 2) if k)
    err2 = _noqual(accumulateTrans([x["subqual"] for x in p1]))
    r = dada2_b200.dada(ds, err=err, pool="pseudo", errorEstimationFunction=_noqual)
    assert r[0]["pseudo_priors"] == rule and V in rule
    assert np.array_equal(r[0]["err_in"], err)
    for d, got in zip(ds, r):
        want = dada2_b200.dada_uniques(d["uniques"], d["abundances"], [s in rule for s in d["uniques"]], err2, d["quals"])
        cases.assert_same(got, want, rtol=0, label="pseudo pass 2")
    assert V in r[2]["denoised"]


def test_learnErrors_stops_after_enough_bases():
    import dada2_b200
    from dada2_b200.errmodel import accumulateTrans
    from dada2_b200 import derep
    d1 = derep.derepFastq(FILES[0])
    b1 = float(np.sum(d1["abundances"] * np.array([len(s) for s in d1["uniques"]])))
    one = dada2_b200.learnErrors(FILES, nbases=b1 - 1)
    assert one["nsamples"] == 1
    two = dada2_b200.learnErrors(FILES, nbases=b1 + 1)
    assert two["nsamples"] == 2
    dds = dada2_b200.dada(_sam(), err=None, selfConsist=True, verbose=False, OMEGA_C=0)
    assert np.array_equal(two["err_out"], dds[0]["err_out"])
    assert np.array_equal(two["trans"], accumulateTrans([x["trans"] for x in dds]))
    assert len(two["err_in"]) == len(dds[0]["err_in"])

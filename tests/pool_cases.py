"""Shared sample-pooling cases (dd_pool.cu, include/dada2b_pool.h) and their check against the host combineDereps2
(dada2_b200.derep.combineDereps2, the restatement of R/multiSample.R:165-203 that tests/test_derep_oracle.py pins).

Each case is (name, dereps, priors): dereps are derep dicts as derepFastq returns them, priors one bool array per sample."""
import os

import numpy as np

from tests import derep_cases as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
NA_INT = np.iinfo(np.int32).min


def sam_dereps():
    from oracle import derep as O
    from dada2_b200 import derep
    return [O.derep_reads(*derep.read_fastq(os.path.join(GOLDEN, f))) for f in ("sam1F.fastq.gz", "sam2F.fastq.gz")]


def hand_derep(seqs, abund, rng, maxlen=None):
    """A derep dict with fractional mean qualities (NaN beyond each length) and a shuffled read -> unique map."""
    maxlen = maxlen or max(len(s) for s in seqs)
    q = np.full((len(seqs), maxlen), np.nan)
    for i, s in enumerate(seqs):
        q[i, :len(s)] = rng.integers(2 * 7, 2 * 41, len(s)) / 2.0 + rng.integers(0, 3, len(s)) / 3.0
    mp = np.repeat(np.arange(1, len(seqs) + 1, dtype=np.int32), abund)
    rng.shuffle(mp)
    return {"uniques": list(seqs), "abundances": np.asarray(abund, np.int32), "quals": q, "map": mp}


def split_dereps(nreads, nsamp, seed, L=60, zero_len=0):
    """derep_cases.synthetic's reads (ragged lengths, proper prefixes, ties) dealt unevenly to nsamp samples."""
    from oracle import derep as O
    s, q = D.synthetic(nreads, seed=seed, L=L, zero_len=zero_len)
    rng = np.random.default_rng(seed)
    who = rng.choice(nsamp, len(s), p=np.arange(1, nsamp + 1) / (nsamp * (nsamp + 1) / 2))
    return [O.derep_reads([s[i] for i in np.flatnonzero(who == k)], [q[i] for i in np.flatnonzero(who == k)]) for k in range(nsamp)]


def _rand_seqs(rng, n, L):
    return ["".join("ACGT"[i] for i in rng.integers(0, 4, L)) for _ in range(n)]


def random_priors(dereps, seed):
    rng = np.random.default_rng(seed)
    return [rng.random(len(d["uniques"])) < 0.2 for d in dereps]


def cases(big=False):
    rng = np.random.default_rng(11)
    out = [("sam1F+sam2F", sam_dereps())]
    out.append(("synthetic split 3", split_dereps(6000 if big else 2500, 3, seed=3)))
    out.append(("synthetic split 5, NA maps", split_dereps(3000, 5, seed=4, zero_len=4)))
    a, b = split_dereps(1500, 1, seed=5, L=50)[0], split_dereps(1500, 1, seed=6, L=72)[0]
    out.append(("maxlen differs per sample", [a, b, a]))
    X, Y, Z, W = _rand_seqs(rng, 4, 40)
    out.append(("pooled ties across samples", [hand_derep([X, Y], [5, 3], rng), hand_derep([Z, Y, W], [4, 2, 5], rng),
                                               hand_derep([W[:33], X[:20]], [5, 5], rng, maxlen=45)]))
    base = _rand_seqs(rng, 30, 55)
    out.append(("one-unique sample", [hand_derep(base[:10], rng.integers(1, 9, 10), rng), hand_derep([base[3]], [7], rng),
                                      hand_derep([base[29]], [1], rng)]))
    same = hand_derep(base[:12], rng.integers(1, 20, 12), rng)
    out.append(("identical samples", [same, same, same]))
    out.append(("disjoint samples", [hand_derep(base[:10], rng.integers(1, 9, 10), rng), hand_derep(base[10:20], rng.integers(1, 9, 10), rng),
                                     hand_derep(base[20:], rng.integers(1, 9, 10), rng)]))
    every = []
    for k in range(6):
        pick = [base[0]] + [base[j] for j in rng.choice(np.arange(1, 30), 8, replace=False)]
        rng.shuffle(pick)
        every.append(hand_derep(pick, rng.integers(1, 30, 9), rng))
    out.append(("a sequence in every sample", every))
    return [(name, ds, random_priors(ds, k)) for k, (name, ds) in enumerate(out)]


def expected(dereps, priors=None):
    """combineDereps2's result (NA map entries restored: the host restatement indexes with them), plus index and prior OR."""
    from dada2_b200.derep import combineDereps2
    safe = []
    for d in dereps:
        m = np.asarray(d["map"]).copy()
        m[m == NA_INT] = 1
        safe.append(dict(d, map=m))
    want = combineDereps2(safe)
    nam = np.concatenate([np.asarray(d["map"]) == NA_INT for d in dereps])
    want["map"][nam] = NA_INT
    pos = {s: i for i, s in enumerate(want["uniques"])}
    want["index"] = np.array([pos[s] + 1 for d in dereps for s in d["uniques"]], np.int32)
    pr = np.zeros(len(pos), bool)
    if priors is not None:
        for d, p in zip(dereps, priors):
            for s, f in zip(d["uniques"], p):
                pr[pos[s]] |= bool(f)
    want["prior"] = pr
    return want


def assert_same(got, want, label="", quals=True):
    assert got["uniques"] == want["uniques"], label + " uniques / order"
    assert np.array_equal(got["abundances"], want["abundances"]), label + " abundances"
    assert np.array_equal(got["map"], want["map"]), label + " map"
    assert np.array_equal(got["index"], want["index"]), label + " index"
    assert np.array_equal(got["prior"], want["prior"]), label + " prior OR"
    if quals:
        a, b = np.asarray(got["quals"]), np.asarray(want["quals"])
        assert a.shape == b.shape and np.array_equal(np.isnan(a), np.isnan(b)), label + " NA pattern"
        fin = ~np.isnan(b)
        assert np.array_equal(a[fin].view(np.uint64), b[fin].view(np.uint64)), label + " pooled means (bit-exact)"
        assert got["qmax"] == np.nanmax(b), label + " qmax"


def check_all(big=False):
    from dada2_b200.derep import pool_dereps
    for name, ds, pr in cases(big):
        got = pool_dereps(ds, priors=pr)
        assert_same(got, expected(ds, pr), name)
        nq = pool_dereps(ds, want_quals=False)
        assert nq["quals"] is None and not nq["prior"].any()
        assert_same(dict(nq, prior=expected(ds)["prior"]), expected(ds), name + " want_quals=False", quals=False)


def check_refusals():
    import pytest
    from dada2_b200 import Dada2bError
    from dada2_b200.derep import pool_dereps
    rng = np.random.default_rng(2)
    ok = hand_derep(_rand_seqs(rng, 3, 30), [3, 2, 1], rng)
    with pytest.raises(Dada2bError, match="No samples"):
        pool_dereps([])
    with pytest.raises(Dada2bError, match="A/C/G/T"):
        pool_dereps([ok, hand_derep(["ACGTNACGTA"], [2], rng)])
    with pytest.raises(Dada2bError, match="one row for each"):
        pool_dereps([ok, dict(ok, quals=ok["quals"][:2])])
    with pytest.raises(Dada2bError, match="as many columns"):
        pool_dereps([ok, dict(ok, quals=ok["quals"][:, :20])])
    with pytest.raises(Dada2bError, match="different lengths"):
        pool_dereps([ok, dict(ok, abundances=ok["abundances"][:2])])
    with pytest.raises(Dada2bError, match="integer range"):
        pool_dereps([dict(ok, abundances=np.array([2 ** 30, 1, 1], np.int32))] * 2 + [ok])
    with pytest.raises(Dada2bError, match="Duplicate"):
        pool_dereps([hand_derep([ok["uniques"][0]] * 2, [1, 1], rng)])
    with pytest.raises(Dada2bError, match="map"):
        pool_dereps([ok, dict(ok, map=np.array([1, 4], np.int32))])

"""Loader of tests/golden/collapse.npz (written by tools/make_golden_collapse.py) and the checks shared by the emulator and
GPU tests of collapseNoMismatch."""
import json
import os

import numpy as np

from tests import collapse_ref as R

HERE = os.path.dirname(os.path.abspath(__file__))
_G = None


def golden():
    global _G
    if _G is None:
        z = np.load(os.path.join(HERE, "golden", "collapse.npz"))
        _G = {k: z[k] for k in z.files}
        _G["meta"] = json.loads(str(_G["meta"]))
    return _G


def table(name):
    g = golden()
    return g[name + "_mat"], [str(c) for c in g[name + "_cols"]], [str(r) for r in g[name + "_rows"]]


def cases():
    return [(k, name, dict(o)) for k, (name, o) in enumerate(golden()["meta"]["cases"])]


def expected(k):
    g = golden()
    return g["c%d_mat" % k], [str(c) for c in g["c%d_cols" % k]]


def pairs(name):
    """-> query-ordered seqs, query index, ref index (every pair j > i)"""
    g = golden()
    return [str(s) for s in g[name + "_seqs"]], g[name + "_pq"], g[name + "_pr"]


def ham(name, vec, band):
    return golden()["%s_ham_v%d_b%d" % (name, int(vec), band)]


def scr(name, m):
    return golden()["%s_scr_m%d" % (name, m)]


def aligners(name):
    return [tuple(a) for a in golden()["meta"]["tables"][name]["aligners"]]


def overlaps(name):
    return golden()["meta"]["tables"][name]["minOverlap"]


def check_tables(collapse_fn, case_ids=None):
    """collapse_fn(mat, cols, **opts) -> (mat, cols); compared with the goldens, matrix and column names."""
    for k, name, o in cases():
        if case_ids is not None and k not in case_ids:
            continue
        mat, cols, _ = table(name)
        m, c = collapse_fn(mat, cols, **o)
        wm, wc = expected(k)
        assert list(c) == wc, (k, name, o)
        assert np.array_equal(np.asarray(m), wm), (k, name, o)


def check_pairs(hook, names=("families", "repeats")):
    """hook(seqs, query, ref, minOverlap, vec, band) -> int32[npairs, 3]; every golden pair, every aligner and screen."""
    for name in names:
        seqs, pq, pr = pairs(name)
        for v, b in aligners(name):
            m0 = overlaps(name)[0]
            out = hook(seqs, pq, pr, m0, bool(v), b)
            want = ham(name, v, b)
            assert np.array_equal(out[:, 2], want), (name, v, b, np.nonzero(out[:, 2] != want)[0][:10])
            assert not np.any((out[:, 1] == 0) & (want == 0)), (name, v, b)          # the filter never rejects a ham-0 pair
            ver = np.array([R.overlap_filter(seqs[j], seqs[i], band=b) for j, i in zip(pq, pr)], np.int32)
            assert np.array_equal(out[:, 1], ver), (name, v, b, np.nonzero(out[:, 1] != ver)[0][:10])   # the verdict, pair by pair
            assert np.array_equal(out[:, 0], scr(name, m0)), (name, m0)
        for m in overlaps(name)[1:]:
            out = hook(seqs, pq, pr, m, True, -1)
            assert np.array_equal(out[:, 0], scr(name, m)), (name, m)
            assert np.array_equal(out[:, 2], ham(name, 1, -1)), (name, m)


def large_table(nfam=500, fam_size=40, genus_size=5, nsamp=96, seed=20):
    """About nfam * fam_size V4-like ASVs (~250 nt) x nsamp samples: genera of genus_size families share their first 20
    bases and ~95 % of the rest; members of a family are its backbone with 1-3 substitutions, truncated or extended ends,
    shifts and single-base indels.  -> (int32 mat [nsamp, nseq], colnames)"""
    rng = np.random.default_rng(seed)

    def rs(n):
        return "".join("ACGT"[i] for i in rng.integers(0, 4, n))

    def mut(s, k, lo=0):
        s = list(s)
        for p in rng.choice(np.arange(lo, len(s)), k, replace=False):
            s[p] = "ACGT"[("ACGT".index(s[p]) + 1 + int(rng.integers(0, 3))) % 4]
        return "".join(s)

    seqs = []
    for f in range(nfam):
        if f % genus_size == 0:
            G = rs(253)
        B = mut(G, 12, lo=20)
        fam = [B]
        while len(fam) < fam_size:
            t = int(rng.integers(0, 12))
            if t < 7: v = mut(B, int(rng.integers(1, 4)))
            elif t == 7: v = B[int(rng.integers(1, 6)):]
            elif t == 8: v = B[:-int(rng.integers(1, 6))] if rng.random() < 0.5 else B + rs(int(rng.integers(1, 5)))
            elif t == 9: k = int(rng.integers(1, 4)); v = B[k:] + rs(k)
            elif t == 10: p = int(rng.integers(30, 220)); v = B[:p] + rs(1) + B[p:]
            else: p = int(rng.integers(30, 220)); v = B[:p] + B[p + 1:]
            fam.append(v)
        seqs += fam
    seqs = list(dict.fromkeys(seqs))
    ab = np.exp(rng.normal(3, 1.5, len(seqs)))
    mat = rng.poisson(ab[None, :] / 8, (nsamp, len(seqs))) * (rng.random((nsamp, len(seqs))) < 0.3)
    mat[int(rng.integers(0, nsamp)), :] += 1
    return mat.astype(np.int32), seqs


def screen_pairs(seqs, m):
    """Every pair (j > i) of seqs passing the prefix screen, all sequences at least m long: -> int32 query, ref arrays"""
    assert all(len(s) >= m for s in seqs)
    by_prefix = {}
    for i, s in enumerate(seqs):
        by_prefix.setdefault(s[:m], []).append(i)
    out = set()
    for j, s in enumerate(seqs):
        for p in range(len(s) - m + 1):
            for i in by_prefix.get(s[p:p + m], ()):
                if i != j:
                    out.add((max(i, j), min(i, j)))
    q, r = (np.array(sorted(out), np.int32).T if out else (np.zeros(0, np.int32), np.zeros(0, np.int32)))
    return q, r

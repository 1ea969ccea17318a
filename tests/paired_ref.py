"""Independent restatement of mergePairs' per-sample R (R/paired.R:111-197) in numpy, for the tests.

Tabulation is np.unique over the (rF, rR) rows with return_index (unique()'s first-occurrence order), NA rows removed after
unique; ordering is a stable argsort of -abundance.  Per-pairing (nmatch, nmismatch, nindel, consensus) come from the
reference's own evaluate.cpp (oracle.ref.merge_pair) when oracle/_ref has it, otherwise from the CPU restatement
(oracle.port.merge_pair).
"""
import numpy as np

NA = np.iinfo(np.int32).min
_COMP = str.maketrans("ACGT", "TGCA")


def rc(s):
    return s.translate(_COMP)[::-1]


_CACHE = {}


def _merge_pair():
    """merge_pair(s1, s2, **opts), memoised: the same pair recurs across samples."""
    from oracle import port, ref
    fn = ref.merge_pair if ref.available() else port.merge_pair

    def mp(s1, s2, **o):
        key = (fn, s1, s2, tuple(sorted(o.items())))
        if key not in _CACHE:
            _CACHE[key] = fn(s1, s2, **o)
        return _CACHE[key]
    return mp


def _lookup(dmap, m):
    m = np.asarray(m, np.int64)
    dmap = np.asarray(dmap, np.int64)
    out = np.full(len(m), NA, np.int64)
    ok = m != NA
    out[ok] = dmap[m[ok] - 1]
    return out


def merge_sample(dadaF, derepF, dadaR, derepR, minOverlap=12, maxMismatch=0, returnRejects=False, propagateCol=(), justConcatenate=False,
                 trimOverhang=False, match=1, mismatch=None, gap=None, homo_gap=None):
    mapF, mapR = np.asarray(derepF["map"]), np.asarray(derepR["map"])

    def mx(m):
        v = m[m != NA]
        return int(v.max()) if len(v) else None
    if not (len(mapF) == len(mapR) and mx(mapF) == len(dadaF["map"]) and mx(mapR) == len(dadaR["map"])):
        raise ValueError("Non-corresponding derep-class and dada-class objects.")
    rF, rR = _lookup(dadaF["map"], mapF), _lookup(dadaR["map"], mapR)
    rows = np.stack([rF, rR], axis=1) if len(rF) else np.zeros((0, 2), np.int64)
    uq, first, counts = np.unique(rows, axis=0, return_index=True, return_counts=True)
    o = np.argsort(first, kind="stable")                          # unique(pairdf): first-occurrence order
    uq, counts = uq[o], counts[o]
    keep = (uq[:, 0] != NA) & (uq[:, 1] != NA)
    uq, counts = uq[keep], counts[keep]
    if len(uq) == 0:
        d = {c: np.zeros(0, np.int32) for c in ("sequence", "abundance", "forward", "reverse", "nmatch", "nmismatch", "nindel", "prefer")}
        d["sequence"], d["accept"] = [], np.zeros(0, bool)
        return d
    fwd, rev = uq[:, 0].astype(np.int32), uq[:, 1].astype(np.int32)
    clF, clR = dadaF["clustering"], dadaR["clustering"]
    Fs = [clF["sequence"][k - 1] for k in fwd]
    Rs = [rc(clR["sequence"][k - 1]) for k in rev]
    n = len(fwd)
    if justConcatenate:
        seq = [f + "NNNNNNNNNN" + r for f, r in zip(Fs, Rs)]
        nm = nmm = nid = np.zeros(n, np.int32)
        prefer = np.full(n, NA, np.int32)
        accept = np.ones(n, bool)
    else:
        sc = -64 if maxMismatch == 0 else -8
        mm = sc if mismatch is None else mismatch
        gp = sc if gap is None else gap
        prefer = (1 + (np.asarray(clR["n0"])[rev - 1] > np.asarray(clF["n0"])[fwd - 1])).astype(np.int32)
        mp = _merge_pair()
        al = [mp(f, r, match=match, mismatch=mm, gap_p=gp, homo_gap_p=homo_gap, prefer=int(p), trim_overhang=bool(trimOverhang))
              for f, r, p in zip(Fs, Rs, prefer)]
        nm = np.array([a["nmatch"] for a in al], np.int32)
        nmm = np.array([a["nmismatch"] for a in al], np.int32)
        nid = np.array([a["nindel"] for a in al], np.int32)
        accept = (nm >= minOverlap) & ((nmm + nid) <= maxMismatch)
        seq = [a["sequence"] for a in al]
    seq = [s if a else "" for s, a in zip(seq, accept)]
    d = {"sequence": seq, "abundance": counts.astype(np.int32), "forward": fwd, "reverse": rev, "nmatch": nm, "nmismatch": nmm,
         "nindel": nid, "prefer": prefer, "accept": accept}
    for col in [c for c in propagateCol if c in clF]:
        d["F." + col] = [clF[col][k - 1] for k in fwd]
        d["R." + col] = [clR[col][k - 1] for k in rev]
    o = np.argsort(-d["abundance"].astype(np.int64), kind="stable")
    d = {k: ([v[i] for i in o] if isinstance(v, list) else v[o]) for k, v in d.items()}
    if not returnRejects:
        a = d["accept"]
        d = {k: ([x for x, ok in zip(v, a) if ok] if isinstance(v, list) else v[a]) for k, v in d.items()}
    return d


def distinct_triples(dadaFs, dadaRs, mergers_all):
    """Distinct (forward sequence, reverse sequence, prefer) over all pairings (mergers with returnRejects=TRUE)."""
    out = set()
    for dF, dR, m in zip(dadaFs, dadaRs, mergers_all):
        for f, r, p in zip(m["forward"], m["reverse"], m["prefer"]):
            out.add((dF["clustering"]["sequence"][f - 1], dR["clustering"]["sequence"][r - 1], int(p)))
    return len(out)


def assert_same(got, want, label=""):
    assert list(got.keys()) == list(want.keys()), (label, list(got.keys()), list(want.keys()))
    for k in want:
        g, w = got[k], want[k]
        if isinstance(w, list):
            assert [x.item() if hasattr(x, "item") else x for x in g] == [x.item() if hasattr(x, "item") else x for x in w], (label, k)
        else:
            assert np.asarray(g).dtype.kind == np.asarray(w).dtype.kind and np.array_equal(np.asarray(g), np.asarray(w)), (label, k, g[:10], w[:10])

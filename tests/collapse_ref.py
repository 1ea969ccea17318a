"""collapseNoMismatch (R/multiSample.R:104-160) restated line for line in Python over a pluggable nwhamming, plus a numpy
restatement of the library's prefix screen and exact overlap filter (DESIGN.md 17).

Parity of the loop itself is unpinned against R (no R here): `collapse` follows the R source statement by statement; the
native part it calls, nwhamming, is the reference's own compiled C++ (`ref_nwhamming`) or the CPU port (`port_nwhamming`).
    vec=TRUE : C_nwvec -> nwalign_vectorized2(query, ref, end_gap 0, band), then mismatch + indel of C_eval_pair.  The
               reference's get_ham_endsfree (chimera.cpp) counts exactly that on the same alignment, so the compiled
               bimera_pair hook with max_shift = band gives it.
    vec=FALSE: C_nwalign(endsfree) -> C_eval_pair, the compiled merge_pair hook (mismatch + indel).
"""
import numpy as np


def ref_nwhamming(s1, s2, vec=True, band=-1, match=5, mismatch=-4, gap=-8):
    from oracle import ref
    if vec:
        return ref.bimera_pair(s1, s2, match=match, mismatch=mismatch, gap_p=gap, max_shift=band)["ham"]
    r = ref.merge_pair(s1, s2, match=match, mismatch=mismatch, gap_p=gap, band=band)
    return r["nmismatch"] + r["nindel"]


def port_nwhamming(s1, s2, vec=True, band=-1, match=5, mismatch=-4, gap=-8):
    from oracle import port
    if vec:
        return port.bimera_pair(s1, s2, match=match, mismatch=mismatch, gap_p=gap, max_shift=band)["ham"]
    r = port.merge_pair(s1, s2, match=match, mismatch=mismatch, gap_p=gap, band=band)
    return r["nmismatch"] + r["nindel"]


def eval_pair(a0, a1):
    """C_eval_pair (evaluate.cpp:73-120) on two aligned strings -> (match, mismatch, indel)."""
    n = len(a0)
    s1g = s2g = True
    start = -1
    while True:
        start += 1
        s1g = s1g and a0[start] == "-"
        s2g = s2g and a1[start] == "-"
        if not ((s1g or s2g) and start < n):
            break
    s1g = s2g = True
    end = n
    while True:
        end -= 1
        s1g = s1g and a0[end] == "-"
        s2g = s2g and a1[end] == "-"
        if not ((s1g or s2g) and end >= start):
            break
    m = x = d = 0
    for i in range(start, end + 1):
        if a0[i] == "-" or a1[i] == "-":
            d += 1
        elif a0[i] == a1[i]:
            m += 1
        else:
            x += 1
    return m, x, d


def substr(s, n):
    """R's substr(s, 1, n): the whole string when it is shorter, "" for n <= 0."""
    return s[:max(n, 0)]


def screen(query, ref, minOverlap):
    """grepl(prefix, ref, fixed=TRUE) || grepl(prefix.ref, query, fixed=TRUE) (:127-131)."""
    return substr(query, minOverlap) in ref or substr(ref, minOverlap) in query


def _codes(s):
    return np.frombuffer(s.encode(), np.uint8)


def overlap_filter(s1, s2, match=5, mismatch=-4, band=-1):
    """The library's filter verdict: True = the pair needs alignment, False = nwhamming(s1, s2) > 0 is proved.
    For each shift s (s1 base i against s2 base i + s): g(s) = match * m(s) + mismatch * x(s); LB = max g; E = some shift
    attaining LB has x = 0; unbanded only, LB > 0 and not E reject."""
    if band >= 0:
        return True
    a, b = _codes(s1), _codes(s2)
    best, exact = None, False
    for s in range(-(len(a) - 1), len(b)):
        lo, hi = max(0, -s), min(len(a), len(b) - s)
        o = hi - lo
        x = int(np.count_nonzero(a[lo:hi] != b[lo + s:hi + s]))
        g = match * (o - x) + mismatch * x
        if best is None or g > best:
            best, exact = g, x == 0
        elif g == best and x == 0:
            exact = True
    return not (best > 0 and not exact)


def _order_desc(v):
    return list(np.argsort(-np.asarray(v, dtype=np.int64), kind="stable"))


def collapse(seqtab, colnames, minOverlap=20, orderBy="abundance", identicalOnly=False, vec=True, band=-1, nwhamming=ref_nwhamming,
             match=5, mismatch=-4, gap=-8):
    """R/multiSample.R:104-160 statement by statement.  -> (int32 mat, colnames)"""
    seqtab = np.asarray(seqtab, dtype=np.int64)
    cols = list(colnames)
    # dupes <- duplicated(colnames(seqtab)); st[,sq] <- st[,sq] + seqtab[,i]   (:106-114)
    seen, keep = {}, []
    for k, sq in enumerate(cols):
        if sq in seen:
            continue
        seen[sq] = len(keep)
        keep.append(k)
    st = seqtab[:, keep].copy()
    kept = set(keep)
    for k, sq in enumerate(cols):
        if k not in kept:
            st[:, seen[sq]] += seqtab[:, k]
    seqtab, cols = st, [cols[k] for k in keep]
    if identicalOnly:
        return seqtab.astype(np.int32), cols
    # unqs.srt <- sort(getUniques(seqtab), decreasing=TRUE); seqs <- names(unqs.srt)   (:118-119)
    seqs = [cols[k] for k in _order_desc(seqtab.sum(axis=0))]
    seqs_out = []
    collapsed = np.zeros(seqtab.shape, np.int64)
    idx = {sq: k for k, sq in enumerate(cols)}
    for query in seqs:                                                   # :125-144
        added = False
        prefix = substr(query, minOverlap)
        for ref in seqs_out:
            prefix_ref = substr(ref, minOverlap)
            if prefix in ref or prefix_ref in query:
                if nwhamming(query, ref, vec=vec, band=band, match=match, mismatch=mismatch, gap=gap) == 0:
                    collapsed[:, idx[ref]] += seqtab[:, idx[query]]
                    added = True
                    break
        if not added:
            collapsed[:, idx[query]] = seqtab[:, idx[query]]
            seqs_out.append(query)
    outset = set(seqs_out)
    k = [i for i, c in enumerate(cols) if c in outset]                   # :145
    collapsed, cols = collapsed[:, k], [cols[i] for i in k]
    if orderBy is not None:                                              # :147-154
        if orderBy == "abundance":
            o = _order_desc(collapsed.sum(axis=0))
            collapsed, cols = collapsed[:, o], [cols[i] for i in o]
        elif orderBy == "nsamples":
            o = _order_desc((collapsed > 0).sum(axis=0))
            collapsed, cols = collapsed[:, o], [cols[i] for i in o]
    o = _order_desc(collapsed.sum(axis=0))                               # :156
    return collapsed[:, o].astype(np.int32), [cols[i] for i in o]


def query_order(seqtab, colnames):
    """The deduplicated sequences in query order (:106-119)."""
    m, c = collapse(seqtab, colnames, identicalOnly=True)
    return [c[k] for k in _order_desc(m.sum(axis=0))]


def greedy(n, zero_pairs):
    """The host resolution of the greedy loop: rep[j] = smallest kept i < j with (j, i) in zero_pairs, else j."""
    rep = list(range(n))
    for j, i in sorted(zero_pairs):
        if rep[j] == j and rep[i] == i:
            rep[j] = i
    return np.asarray(rep, np.int32)

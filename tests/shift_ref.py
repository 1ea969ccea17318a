"""isShiftDenovo (R/chimeras.R:380-421) restated line for line in Python over a pluggable nwalign, plus a numpy
restatement of the library's overlap filter in its isShiftDenovo form (DESIGN.md 24).

The loop follows the R source statement by statement over a pluggable counts(sq, par) = C_eval_pair(nwalign(sq, par,
band=-1)); by default nwalign is the reference's own compiled nwalign_endsfree (`ref_nwalign`, oracle/_ref) and
C_eval_pair is collapse_ref.eval_pair.
"""
import numpy as np

from tests.collapse_ref import _codes, eval_pair


def ref_nwalign(s1, s2):
    from oracle import ref
    return ref.align(s1, s2, band=-1, mode=1)                   # C_nwalign -> nwalign_endsfree (evaluate.cpp:40-41)


def is_acgt(s):
    return all(c in "ACGT" for c in s)


def shifted_pair_counts(sq1, sq2, nwalign=ref_nwalign):
    """:407-408: al <- nwalign(sq1, sq2, band=-1); C_eval_pair(al[1], al[2]) -> (match, mismatch, indel)."""
    if not (is_acgt(sq1) and is_acgt(sq2)):
        raise ValueError("Sequences must contain only A/C/G/T characters.")          # R/misc.R:186-188
    return eval_pair(*nwalign(sq1, sq2))


def is_shifted_pair(sq1, sq2, minOverlap=20, flagSubseqs=False, counts=shifted_pair_counts):
    """:406-411; counts(sq1, sq2) -> C_eval_pair(nwalign(sq1, sq2, band=-1))"""
    m, x, d = counts(sq1, sq2)
    return (m < len(sq1) or flagSubseqs) and (m < len(sq2) or flagSubseqs) and m >= minOverlap and x == 0 and d == 0


def is_shift(sq, pars, minOverlap=20, flagSubseqs=False, counts=shifted_pair_counts):
    """:413-415 (sapply, then any: every parent is aligned)"""
    return any([is_shifted_pair(sq, par, minOverlap=minOverlap, flagSubseqs=flagSubseqs, counts=counts) for par in pars])


def is_shift_denovo(unqs, minOverlap=20, flagSubseqs=False, counts=shifted_pair_counts):
    """:384-400 over a {sequence: abundance} dict (getUniques' result) -> {sequence: flag}.  flagSubseqs is not passed on
    (:391)."""
    abunds = list(unqs.values())
    seqs = list(unqs.keys())

    def loop_fun(sq, abund):
        pars = [s for s, a in zip(seqs, abunds) if a > abund]
        if len(pars) == 0:
            return False
        return is_shift(sq, pars, minOverlap=minOverlap, counts=counts)

    shifts = [loop_fun(sq, a) for sq, a in zip(seqs, abunds)]
    return {sq: bool(f) for sq, f in zip(seqs, shifts)}


def directed_pairs(seqs, abunds):
    """Every (query, parent) pair R aligns: abund[parent] > abund[query], both non-empty -> int32 query, parent"""
    ab = np.asarray(abunds, np.int64)
    q, p = np.nonzero(ab[:, None] < ab[None, :])
    keep = np.array([bool(seqs[i]) and bool(seqs[j]) for i, j in zip(q, p)], bool) if len(q) else np.zeros(0, bool)
    return q[keep].astype(np.int32), p[keep].astype(np.int32)


def screen(sq, par, minOverlap):
    """The prefix screen the library applies: grepl(prefix(sq), par) || grepl(prefix(par), sq), every pair for m <= 0."""
    if minOverlap <= 0:
        return True
    return sq[:minOverlap] in par or par[:minOverlap] in sq


def shift_filter(s1, s2, minOverlap=20, match=5, mismatch=-4):
    """The library's filter verdict: True = the pair needs alignment, False = it is proved not to be a shift.
    g(s) = match * m(s) + mismatch * x(s) over every shift with overlap o(s) > 0; LB = max g; E = some shift attaining LB has
    x = 0 and o in [max(minOverlap, 1), min(l1, l2) - 1]; LB > 0 and not E reject."""
    a, b = _codes(s1), _codes(s2)
    lo_o, hi_o = max(minOverlap, 1), min(len(a), len(b)) - 1
    best, exact = None, False
    for s in range(-(len(a) - 1), len(b)):
        lo, hi = max(0, -s), min(len(a), len(b) - s)
        o = hi - lo
        x = int(np.count_nonzero(a[lo:hi] != b[lo + s:hi + s]))
        g = match * (o - x) + mismatch * x
        ex = x == 0 and lo_o <= o <= hi_o
        if best is None or g > best:
            best, exact = g, ex
        elif g == best and ex:
            exact = True
    return not (best > 0 and not exact)

"""Restatement of removePrimers (R/filter.R:81-233) with allow.indels=FALSE, for the tests.

Biostrings is not part of the reference, so the matcher below restates Biostrings' naive inexact matcher (which
vmatchPattern(..., with.indels=FALSE) uses) from its definition; parity with Biostrings itself is unpinned.  Every rule
of DESIGN.md 19 is stated once here:

  1. letters: fixed = C_isACGT(primer).  fixed: a primer letter matches only the same read letter.  Otherwise letters
     match when their IUPAC base sets intersect, both ways (N in the read matches anything).
  2. placements: the primer's first letter goes at every 0-based shift from min_shift = (P <= k ? 1 - P : -k) while its
     end stays <= L - min_shift; a primer letter outside the read is a mismatch; <= k mismatches is a hit at 1-based
     [shift + 1, shift + P]; hits are listed by increasing start.
  3. four scans: each primer against the read and against reverseComplement(read) (qualities reversed).
  4. several hits: the first forward hit and the last reverse hit are used.
  5. flip = orient & no forward hit as read & a forward hit on the reverse complement; the flipped read replaces the read
     in place (output order = input order).
  6. whole-file skip: no read has a forward hit as read, or (with a reverse primer) none has a reverse hit as read;
     checked before flipping.
  7. keep: a forward hit and (with a reverse primer) a reverse hit; first = end(fwd) + 1 if trim_fwd else 1; last =
     start(rev) - 1 if trim_rev and a reverse primer else L; kept only if last > first; narrowed to [first, last].
"""
import numpy as np

IUPAC = "ACGTRYSWKMBDHVN"
MASK = {"A": 1, "C": 2, "G": 4, "T": 8, "R": 5, "Y": 10, "S": 6, "W": 9, "K": 12, "M": 3, "B": 14, "D": 13, "H": 11, "V": 7, "N": 15}
_COMP = str.maketrans("ACGTRYKMBVDHSWN", "TGCAYRMKVBHDSWN")
_MASK_LUT = np.zeros(256, np.uint8)
for _c, _m in MASK.items():
    _MASK_LUT[ord(_c)] = _m
_SINGLE = np.zeros(256, np.uint8)
for _c in "ACGT":
    _SINGLE[ord(_c)] = MASK[_c]

KEPT, NO_FWD, NO_REV, EMPTY, SKIPPED = 0, 1, 2, 3, 4
FLIPPED, MULTI_FWD, MULTI_REV = 1, 2, 4


def rc(s):
    return s[::-1].translate(_COMP)


def is_acgt(p):                                                    # C_isACGT (src/evaluate.cpp:184)
    return all(c in "ACGT" for c in p)


def min_shift(P, k):
    return 1 - P if P <= k else -k


# ---- rule 1 + 2, literally -------------------------------------------------------------------------------------------
def letters_match(p, s, fixed):
    if fixed:
        return p == s
    return (MASK[p] & MASK[s]) != 0


def mismatches_at(P, S, shift, fixed):
    n = 0
    for i, p in enumerate(P):
        j = shift + i
        if j < 0 or j >= len(S) or not letters_match(p, S[j], fixed):
            n += 1
    return n


def match_literal(P, S, k):
    """-> [(start, end)] 1-based, by increasing start: the per-shift definition."""
    fixed = is_acgt(P)
    ms = min_shift(len(P), k)
    out = []
    shift = ms
    while shift + len(P) <= len(S) - ms:
        if mismatches_at(P, S, shift, fixed) <= k:
            out.append((shift + 1, shift + len(P)))
        shift += 1
    return out


# ---- the same, vectorised ---------------------------------------------------------------------------------------------
def match_vec(P, S, k):
    """match_literal with numpy: the read's IUPAC masks (single bases only for a fixed primer), padded with -min_shift
    letters that match nothing at both ends, against the primer's masks at every window."""
    P_len = len(P)
    pad = -min_shift(P_len, k)
    lut = _SINGLE if is_acgt(P) else _MASK_LUT
    s = lut[np.frombuffer(S.encode(), np.uint8)] if S else np.zeros(0, np.uint8)
    padded = np.concatenate([np.zeros(pad, np.uint8), s, np.zeros(pad, np.uint8)])
    if len(padded) < P_len:
        return []
    pm = _MASK_LUT[np.frombuffer(P.encode(), np.uint8)]
    win = np.lib.stride_tricks.sliding_window_view(padded, P_len)
    mism = P_len - ((win & pm[None, :]) != 0).sum(axis=1)
    idx = np.nonzero(mism <= k)[0]
    return [(int(i) - pad + 1, int(i) - pad + P_len) for i in idx]


def summary(hits):
    """-> (count, first_start, first_end, last_start, last_end), zeros without a hit (the hook's record)."""
    if not hits:
        return (0, 0, 0, 0, 0)
    return (len(hits),) + hits[0] + hits[-1]


def scans(seq, pf, pr, k, matcher=match_vec):
    """Rule 3: the four scans of one read, each as summary(): fwd on read, rev on read, fwd on rc(read), rev on rc(read)."""
    r = rc(seq)
    z = (0, 0, 0, 0, 0)
    return [summary(matcher(pf, seq, k)), summary(matcher(pr, seq, k)) if pr is not None else z,
            summary(matcher(pf, r, k)), summary(matcher(pr, r, k)) if pr is not None else z]


# ---- rules 4-7 ----------------------------------------------------------------------------------------------------------
def remove_primers(records, pf, pr=None, k=2, trim_fwd=True, trim_rev=True, orient=True):
    """records: [(seq, quals)] of one file.  -> dict(skipped, multi, reason, flags, out=[(src, seq, quals)])."""
    n = len(records)
    has_rev = pr is not None
    H = [scans(s, pf, pr, k) for s, _ in records]
    hits_fwd = np.array([h[0][0] for h in H], np.int64)
    hits_rev = np.array([h[1][0] for h in H], np.int64)
    reason = np.zeros(n, np.uint8)
    flags = np.zeros(n, np.uint8)
    if hits_fwd.sum() == 0 or (has_rev and hits_rev.sum() == 0):          # rule 6, :157-158
        reason[:] = SKIPPED
        return dict(skipped=True, multi=False, reason=reason, flags=flags, out=[])
    multi = bool(np.any(hits_fwd > 1) or (has_rev and np.any(hits_rev > 1)))
    if orient:
        multi |= any(h[2][0] > 1 or (has_rev and h[3][0] > 1) for h in H)
    out = []
    for i, (s, q) in enumerate(records):
        h = H[i]
        flip = orient and h[0][0] == 0 and h[2][0] > 0                   # rule 5
        if flip:
            s, q = rc(s), list(q)[::-1]
        hf, hr = (h[2], h[3]) if flip else (h[0], h[1])
        fl = (FLIPPED if flip else 0) | (MULTI_FWD if hf[0] > 1 else 0) | (MULTI_REV if has_rev and hr[0] > 1 else 0)
        flags[i] = fl
        if hf[0] == 0:                                                    # rule 7
            reason[i] = NO_FWD
            continue
        if has_rev and hr[0] == 0:
            reason[i] = NO_REV
            continue
        first = hf[2] + 1 if trim_fwd else 1                              # rule 4: the first forward hit's end
        last = hr[3] - 1 if (has_rev and trim_rev) else len(s)            # rule 4: the last reverse hit's start
        if not last > first:
            reason[i] = EMPTY
            continue
        out.append((i, s[first - 1:last], [int(x) for x in list(q)[first - 1:last]]))
    return dict(skipped=False, multi=multi, reason=reason, flags=flags, out=out)


def fastq_bytes(ids, seqs, quals):
    return b"".join(b"@%s\n%s\n+\n%s\n" % (i, s.encode(), bytes(int(x) + 33 for x in q)) for i, s, q in zip(ids, seqs, quals))


def vector_decide(hits, lens, has_rev, trim_fwd=True, trim_rev=True, orient=True):
    """Rules 4-7 vectorised over hook records (HIT_DTYPE [n, 4]) of a file that is not skipped; lens: read lengths.
    -> (reason, flags) as dada2b_remove_primers defines them."""
    c = hits["count"]
    flip = orient & (c[:, 0] == 0) & (c[:, 2] > 0)
    hf_c, hr_c = np.where(flip, c[:, 2], c[:, 0]), np.where(flip, c[:, 3], c[:, 1])
    first = np.where(flip, hits["first_end"][:, 2], hits["first_end"][:, 0]) + 1 if trim_fwd else np.ones(len(c), np.int64)
    last = np.where(flip, hits["last_start"][:, 3], hits["last_start"][:, 1]) - 1 if (has_rev and trim_rev) else np.asarray(lens)
    reason = np.full(len(c), KEPT, np.uint8)
    reason[~(last > first)] = EMPTY
    if has_rev:
        reason[hr_c == 0] = NO_REV
    reason[hf_c == 0] = NO_FWD
    flags = np.where(flip, FLIPPED, 0) | np.where(hf_c > 1, MULTI_FWD, 0) | np.where(has_rev & (hr_c > 1), MULTI_REV, 0)
    return reason, flags.astype(np.uint8)

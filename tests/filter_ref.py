"""Line-by-line restatement of the reference's read filter (R/filter.R), for the tests only.

fastqFilter (:613-730) and fastqPairedFilter (:878-1141) per FastqStreamer chunk of n reads, stages 1-12 in the R order,
plus C_matchRef / C_matrixEE (src/filter.cpp) and seqComplexity / sindex (:1248-1275) with the sum sequential in
np.longdouble, as R's rsum adds on x86-64.  Parity of the R-level logic is not pinned against R itself (no R here), as for
derep and collapse; C_matchRef and C_matrixEE are pinned against the compiled reference where oracle/_ref is built.

Reason codes: 0 kept, else the first stage that removed the read (pair); mate bits 1/2 say which mate failed that stage
(every mate whose predicate fails there), bit 4 that orient.fwd flipped the read / swapped the pair.
"""
import ctypes as C
import math
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EE_TAB = [math.pow(10.0, -q / 10.0) for q in range(94)]          # C's pow, as C_matrixEE calls it
_COMP = str.maketrans("ACGTRYKMBVDHSWN", "TGCAYRMKVBHDSWN")
INF = math.inf


def rc(s):
    return s.translate(_COMP)[::-1]


def match_ref(seqs, ref, w, non_overlapping):
    """C_matchRef (src/filter.cpp:7-32), including the j += w then j++ skip."""
    r = ref + ref[:w]
    ph = {r[i:i + w] for i in range(len(ref))}
    out = []
    for s in seqs:
        n, j, L = 0, 0, len(s)
        if L >= w:
            while j <= L - w:
                if s[j:j + w] in ph:
                    n += 1
                    if non_overlapping:
                        j += w
                j += 1
        out.append(n)
    return np.array(out, np.int32)


def matrix_ee(q):
    """C_matrixEE for one read: pow(10, -q/10) added in ascending position order."""
    ee = 0.0
    for x in q:
        ee += EE_TAB[int(x)]
    return ee


def tree_ee(q):
    """A pairwise (tree) sum of the same terms -- what a reordered sum would give."""
    t = [EE_TAB[int(x)] for x in q]
    if not t:
        return 0.0
    while len(t) > 1:
        t = [t[i] + t[i + 1] if i + 1 < len(t) else t[i] for i in range(0, len(t), 2)]
    return t[0]


def kmer_counts(s, k):
    cnt = [0] * (4 ** k)
    code = {"A": 0, "C": 1, "G": 2, "T": 3}
    for i in range(len(s) - k + 1):
        w = s[i:i + k]
        if all(c in code for c in w):
            x = 0
            for c in w:
                x = x * 4 + code[c]
            cnt[x] += 1
    return cnt


def sindex(x):
    """exp(sum(-y*log(y))), y = x/sum(x), y > 0; the sum in long double.  NaN for R's NA (sum(x) == 0)."""
    tot = sum(x)
    if tot == 0:
        return math.nan
    s = np.longdouble(0)
    for c in x:
        if c:
            y = c / tot
            s += np.longdouble(-y * math.log(y))
    return math.exp(float(s))


def complexity(s, k=2):
    return sindex(kmer_counts(s, k))


class Opts:
    """One mate's options with the reference's defaults (filterAndTrim)."""

    def __init__(self, truncQ=2, truncLen=0, trimLeft=0, trimRight=0, maxLen=INF, minLen=20, maxN=0, minQ=0, maxEE=INF, rm_phix=True,
                 rm_lowcomplex=0):
        self.truncQ, self.truncLen, self.trimLeft, self.trimRight = truncQ, truncLen, trimLeft, trimRight
        self.maxLen, self.minLen, self.maxN, self.minQ, self.maxEE = maxLen, minLen, maxN, minQ, maxEE
        self.rm_phix, self.rm_lowcomplex = rm_phix, rm_lowcomplex
        self.start = max(1, trimLeft + 1)
        end = truncLen
        self.end = None if end < self.start else end - self.start + 1

    def kw(self):
        return dict(truncQ=self.truncQ, truncLen=self.truncLen, trimLeft=self.trimLeft, trimRight=self.trimRight, maxLen=self.maxLen,
                    minLen=self.minLen, maxN=self.maxN, minQ=self.minQ, maxEE=self.maxEE, rm_phix=self.rm_phix,
                    rm_lowcomplex=self.rm_lowcomplex)


class FilterError(Exception):
    pass


def n_other(s):
    return sum(1 for c in s if c not in "ACGT")


def is_phix(s, phix):
    return match_ref([s], phix, 16, True)[0] >= 2 or match_ref([s], rc(phix), 16, True)[0] >= 2


def _trunc_q(seq, q, tq):
    for p, x in enumerate(q):
        if x <= tq:
            return seq[:p], q[:p]
    return seq, q


def filter_chunks(reads, opts, orient_fwd=None, phix=None, n=100000):
    """reads: list of tuples of mates, each mate (seq, list of int quals); opts: list of Opts per mate.
    -> (reason int[nreads], flags int[nreads], out: list of (src, [(seq, qual) per mate]))."""
    nm = len(opts)
    N = len(reads)
    for o in opts:
        if not (0 <= o.truncQ <= 93):
            raise FilterError("Encoding for this truncQ value not found.")
    reason = [0] * N
    flags = [0] * N
    out = []
    chunk = int(n) if n > 0 else max(N, 1)
    for c0 in range(0, N, chunk):
        # records: [src, flipped, [ [seq, qual], ... per mate ]]
        recs = [[i, 0, [[reads[i][m][0], list(reads[i][m][1])] for m in range(nm)]] for i in range(c0, min(N, c0 + chunk))]

        def drop(stage, pred):                       # pred(rec) -> list of failing mates; remove if any
            nonlocal recs
            keep = []
            for r in recs:
                bad = pred(r)
                if any(bad):
                    reason[r[0]] = stage
                    flags[r[0]] = (4 if r[1] else 0) | sum(1 << m for m in range(nm) if bad[m])
                else:
                    keep.append(r)
            recs = keep

        # 1. orient.fwd
        if orient_fwd is not None:
            if any(c not in "ACGT" for c in orient_fwd):
                raise FilterError("Non-ACGT characters detected in orient.fwd")
            bl = len(orient_fwd)
            if any(len(m[0]) < bl for r in recs for m in r[2]):
                raise FilterError("narrow: a read is shorter than orient.fwd")
            fw, fl = [], []
            for r in recs:
                if nm == 1:
                    s, q = r[2][0]
                    if s[:bl] == orient_fwd:
                        fw.append(r)
                    elif rc(s)[:bl] == orient_fwd:
                        r[1] = 1
                        r[2][0] = [rc(s), q[::-1]]
                        fl.append(r)
                    else:
                        reason[r[0]], flags[r[0]] = 1, 1
                else:
                    if r[2][0][0][:bl] == orient_fwd:
                        fw.append(r)
                    elif r[2][1][0][:bl] == orient_fwd:
                        r[1] = 1
                        r[2] = [r[2][1], r[2][0]]
                        fl.append(r)
                    else:
                        reason[r[0]], flags[r[0]] = 1, 3
            recs = fw + fl
        # 2. maxLen
        drop(2, lambda r: [len(r[2][m][0]) > opts[m].maxLen for m in range(nm)])
        # 3. trimLeft
        drop(3, lambda r: [len(r[2][m][0]) < opts[m].start for m in range(nm)])
        for r in recs:
            for m in range(nm):
                s, q = r[2][m]
                r[2][m] = [s[opts[m].start - 1:], q[opts[m].start - 1:]]
        # 4. trimRight
        drop(4, lambda r: [opts[m].trimRight > 0 and len(r[2][m][0]) <= opts[m].trimRight for m in range(nm)])
        for r in recs:
            for m in range(nm):
                if opts[m].trimRight > 0:
                    s, q = r[2][m]
                    r[2][m] = [s[:len(s) - opts[m].trimRight], q[:len(q) - opts[m].trimRight]]
        # 5. truncQ (trimTails k = 1; width 0 dropped)
        for r in recs:
            for m in range(nm):
                r[2][m] = list(_trunc_q(r[2][m][0], r[2][m][1], opts[m].truncQ))
        drop(5, lambda r: [len(r[2][m][0]) == 0 for m in range(nm)])
        # 6. truncLen
        drop(6, lambda r: [opts[m].end is not None and len(r[2][m][0]) < opts[m].end for m in range(nm)])
        for r in recs:
            for m in range(nm):
                if opts[m].end is not None:
                    s, q = r[2][m]
                    r[2][m] = [s[:opts[m].end], q[:opts[m].end]]
        # 7. minLen
        drop(7, lambda r: [len(r[2][m][0]) < opts[m].minLen for m in range(nm)])
        # 8. maxN (.nFilter: every letter other than A/C/G/T)
        drop(8, lambda r: [n_other(r[2][m][0]) > opts[m].maxN for m in range(nm)])
        # 9. minQ, only when minQ > truncQ;  10. maxEE, only when finite
        drop(9, lambda r: [opts[m].minQ > opts[m].truncQ and not (min(r[2][m][1]) > opts[m].minQ) for m in range(nm)])
        drop(10, lambda r: [opts[m].maxEE < INF and matrix_ee(r[2][m][1]) > opts[m].maxEE for m in range(nm)])
        # 11. rm.phix on the tested mates
        if any(o.rm_phix for o in opts):
            drop(11, lambda r: [bool(opts[m].rm_phix) and is_phix(r[2][m][0], phix) for m in range(nm)])
        # 12. rm.lowcomplex: `> 0` single-end, used as a logical when paired; NA | TRUE is TRUE, otherwise NA stops R
        on = [(o.rm_lowcomplex > 0) if nm == 1 else (o.rm_lowcomplex != 0) for o in opts]
        if any(on):
            keep = []
            for r in recs:
                low = []
                for m in range(nm):
                    if not on[m]:
                        low.append(False)
                        continue
                    cx = complexity(r[2][m][0])
                    low.append(None if math.isnan(cx) else cx < opts[m].rm_lowcomplex)
                if any(x is True for x in low):
                    reason[r[0]] = 12
                    flags[r[0]] = (4 if r[1] else 0) | sum(1 << m for m in range(nm) if low[m] is True)
                elif any(x is None for x in low):
                    raise FilterError("seqComplexity is NA")
                else:
                    keep.append(r)
            recs = keep
        for r in recs:
            flags[r[0]] = 4 if r[1] else 0
            out.append((r[0], [(s, list(q)) for s, q in r[2]]))
    return np.array(reason, np.uint8), np.array(flags, np.uint8), out


def stage_values(seq, q, o, orient_fwd=None, phix=None):
    """What the stage hook reports for one read: (trim_fail, flipped, start, end, n_other, min_q, ee, hits_f, hits_r,
    complexity) on the trim window, whatever stages 8-12 decide."""
    flip = 0
    if orient_fwd is not None:
        bl = len(orient_fwd)
        if seq[:bl] == orient_fwd:
            pass
        elif rc(seq)[:bl] == orient_fwd:
            seq, q, flip = rc(seq), list(q)[::-1], 1
        else:
            return (1, 0, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
    L = len(seq)
    if o.maxLen < INF and L > o.maxLen:
        return (2, flip, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
    if L < o.start:
        return (3, flip, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
    s0, e = o.start - 1, L
    if o.trimRight > 0:
        if e - s0 <= o.trimRight:
            return (4, flip, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
        e -= o.trimRight
    for p in range(s0, e):
        if q[p] <= o.truncQ:
            e = p
            break
    if e == s0:
        return (5, flip, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
    if o.end is not None:
        if e - s0 < o.end:
            return (6, flip, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
        e = s0 + o.end
    if e - s0 < o.minLen:
        return (7, flip, 0, 0, 0, 0, 0.0, 0, 0, 0.0)
    w, wq = seq[s0:e], list(q)[s0:e]
    hf = int(match_ref([w], phix, 16, True)[0]) if phix else 0
    hr = int(match_ref([w], rc(phix), 16, True)[0]) if phix else 0
    return (0, flip, s0, e, n_other(w), min(wq), matrix_ee(wq), hf, hr, complexity(w))


def fastq_bytes(ids, seqs, quals):
    """writeFastq's byte format: @id / sequence / + / quality (Phred+33)."""
    return b"".join(b"@" + i + b"\n" + s.encode() + b"\n+\n" + bytes(int(x) + 33 for x in q) + b"\n" for i, s, q in zip(ids, seqs, quals))


# ---- the compiled reference (oracle/_ref/libdada2ref_filter.so, built by oracle/filter.mk) ----------------------------
_REF = os.path.join(ROOT, "oracle", "_ref", "libdada2ref_filter.so")
_RL = None


def ref_lib():
    global _RL
    if _RL is None and os.path.exists(_REF):
        L = C.CDLL(_REF)
        L.ref_match_ref.argtypes = [C.c_int, C.c_char_p, C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_void_p]
        L.ref_matrix_ee.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _RL = L
    return _RL


def _pack(seqs):
    off = np.zeros(len(seqs) + 1, np.int64)
    np.cumsum([len(s) for s in seqs], out=off[1:])
    return "".join(seqs).encode(), off


def ref_match_ref(seqs, ref, w, non_overlapping):
    buf, off = _pack(seqs)
    hits = np.zeros(max(len(seqs), 1), np.int32)
    ref_lib().ref_match_ref(len(seqs), buf, off.ctypes.data, ref.encode(), int(w), int(bool(non_overlapping)), hits.ctypes.data)
    return hits[:len(seqs)]


def ref_matrix_ee(quals):
    off = np.zeros(len(quals) + 1, np.int64)
    np.cumsum([len(q) for q in quals], out=off[1:])
    q = np.concatenate([np.asarray(x, np.uint8) for x in quals]) if quals else np.zeros(1, np.uint8)
    q = np.ascontiguousarray(q if len(q) else np.zeros(1, np.uint8))
    ee = np.zeros(max(len(quals), 1), np.float64)
    ref_lib().ref_matrix_ee(len(quals), q.ctypes.data, off.ctypes.data, ee.ctypes.data)
    return ee[:len(quals)]

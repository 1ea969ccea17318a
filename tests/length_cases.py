"""Inputs at real amplicon lengths for the steps around dada() -- mergePairs' alignment, bimera detection,
collapseNoMismatch, derepFastq and filterAndTrim -- and cases on both sides of every length-driven layout switch of their
kernels.

Three regimes, each from a seed:
  * MiSeq 2 x 300: 400-480 nt amplicons, forward / reverse reads that overlap by 120-200 nt, with substitutions and
    indels inside the overlap and homopolymer runs;
  * V3-V4 tables: 400-460 nt ASVs (parents, bimeras, one-offs, shifted and truncated copies, tied abundances);
  * PacBio full-length 16S: 1400-1600 nt, CCS qualities up to 93.

Every threshold below is computed from the same formula as the host code that applies it (the function names say
where), never written down as a number, so a later change of a threshold in the host code shows up here as a failing
"the two sides fall in different classes" assertion instead of quietly leaving one side untested.
"""
import numpy as np

NT = "ACGT"


# ---------------------------------------------------------------------------------------------------------------------
# The host formulas
# ---------------------------------------------------------------------------------------------------------------------
def _layout_words(maxlen, minlen, band):
    lbmax = maxlen if band < 0 else min(band + (maxlen - minlen), maxlen)
    wmax = 2 * lbmax + 1
    nchunk = (((wmax + 1) >> 1) + 31) >> 5
    seq_bytes = (maxlen + 15) & ~15
    h_words = (wmax + 2 + 3) & ~3
    ops_words = ((2 * maxlen) // 16 + 2 + 3) & ~3
    mask_words = ((2 * maxlen + 31) // 32 + 2 + 3) & ~3
    ptr_words = (2 * maxlen + 2) * 2 * nchunk
    base = 2 * (seq_bytes // 4) + h_words + ops_words + 3 * mask_words
    return base, ptr_words


def nw_layout(maxlen, minlen, band):
    """nw_warp's per-warp layout of one batch, as planned by dada2b_merge_pairs (dd_merge.cu), plan_align (dd_collapse.cu)
    and setup_align (dd_bimera.cu): four warps per block; the move matrix stays in shared memory while
    16 * (base_words + ptr_words) <= 96 KB, otherwise it goes to per-warp global scratch; beyond 200 KB of shared memory
    the call is refused.  -> "smem", "global" or "refused"."""
    base, ptr = _layout_words(maxlen, minlen, band)
    if 16 * (base + ptr) <= 96 * 1024:
        return "smem"
    return "global" if 16 * base <= 200 * 1024 else "refused"


def first_len(pred, lo=1, hi=20000):
    """The smallest length in [lo, hi) at which pred(length) holds; pred must be monotone over the range."""
    assert not pred(lo) and pred(hi - 1)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if pred(mid):
            hi = mid
        else:
            lo = mid
    return hi


def scratch_switch(band, spread=0):
    """The smallest batch maxlen (minlen = maxlen - spread) whose move matrix no longer fits shared memory."""
    return first_len(lambda L: nw_layout(L, L - spread, band) != "smem", lo=max(2, spread + 1))


def nw_refusal(band, spread=0):
    return first_len(lambda L: nw_layout(L, L - spread, band) == "refused", lo=max(2, spread + 1))


# bimera: k_bimfwd16 (dd_bimfwd16.cu), k_bimfwd (dd_bimfwd.cu), k_bim_align (dd_bimera.cu)
B16_NEG = -16000
SLOT_CLASSES = ((40, 4, 10), (48, 8, 6), (64, 8, 8), (128, 16, 8), (256, 32, 8))      # pick / pick16: (bound, G, ND)


def bim16_worst(maxlen, match, mismatch, gap):
    """launch_bimfwd16's bound on |score|; the kernel runs only while it stays below -B16_NEG / 2."""
    return maxlen * max(abs(mismatch), abs(match)) + abs(gap) + 16


def bim16_fits(maxlen, match=5, mismatch=-4, gap=-8):
    return bim16_worst(maxlen, match, mismatch, gap) < -B16_NEG // 2


def bim16_maxlen(match=5, mismatch=-4, gap=-8):
    """The longest batch maxlen the 16-bit kernel takes at these scores."""
    return first_len(lambda L: not bim16_fits(L, match, mismatch, gap)) - 1


def bim_slots(maxlen, minlen, max_shift):
    """setup_align's fwd_slots: the band width the register kernels must hold for the batch's widest job."""
    lbmax = min(max_shift + (maxlen - minlen), maxlen)
    return ((lbmax + 1) & ~1) + lbmax + 1


def bim_class(slots):
    for bound, g, nd in SLOT_CLASSES:
        if slots <= bound:
            return bound, g, nd
    return None


def bim_route(maxlen, minlen, max_shift=16, match=5, mismatch=-4, gap=-8, mode=2):
    """The first kernel launch_align tries for a batch under DADA2B_BIMFWD=mode: "k_bimfwd16", "k_bimfwd" or
    "k_bim_align" (each later kernel takes what the earlier one hands over)."""
    if mode >= 1 and max_shift >= 0:
        c = bim_class(bim_slots(maxlen, minlen, max_shift))
        if c is not None:
            _, g, _ = c
            ppw = 32 // g
            seq_words = ((maxlen + 15) & ~15) // 4
            mask_words = ((2 * maxlen + 31) // 32 + 2 + 3) & ~3
            if mode == 2 and bim16_fits(maxlen, match, mismatch, gap) and 16 * ppw * (3 * seq_words + 12 * mask_words) <= 160 * 1024:
                return "k_bimfwd16"
            if 16 * ppw * (2 * seq_words + 6 * mask_words) <= 160 * 1024:
                return "k_bimfwd"
    return "k_bim_align"


def slot_spreads(max_shift=16):
    """For each slot class bound: (bound, the largest length spread that stays in it, the smallest that leaves it)."""
    out = []
    for bound, _, _ in SLOT_CLASSES:
        d = first_len(lambda x: bim_slots(2000, 2000 - x, max_shift) > bound, lo=0, hi=1000)
        out.append((bound, d - 1, d))
    return out


# collapseNoMismatch with vec=TRUE: check_opts (dd_collapse.cu)
def vec_fits(maxlen, match=5, mismatch=-4, gap=-8):
    a = max(abs(match), abs(mismatch))
    return a * maxlen + max(a, abs(gap)) <= 32767 and abs(gap) <= 32767


def vec_maxlen(match=5, mismatch=-4, gap=-8):
    return first_len(lambda L: not vec_fits(L, match, mismatch, gap), hi=100000) - 1


VEC_REFUSAL = "too long for the vectorized aligner"


# derep (dd_derep.cu): 16 bases per key word, lengths below SEQLEN = 9999 (the reference's dada.h)
SEQLEN = 9999
DEREP_REFUSAL = "Input sequences exceed the maximum allowed string length."


def derep_key_words(maxlen):
    return (maxlen + 15) // 16


DEREP_LENGTHS = (15, 16, 17, 31, 32, 33, 300, 1500, SEQLEN - 1)


# ---------------------------------------------------------------------------------------------------------------------
# Sequences
# ---------------------------------------------------------------------------------------------------------------------
def rand_seq(rng, n, homo=0.02):
    """n random bases with homopolymer runs of 4-9 nt starting at about `homo` of the positions."""
    s = rng.integers(0, 4, n)
    for p in np.nonzero(rng.random(n) < homo)[0]:
        s[p:p + int(rng.integers(4, 10))] = s[p]
    return "".join(NT[x] for x in s)


def substitute(rng, s, k, lo=0, hi=None):
    s = list(s)
    hi = len(s) if hi is None else hi
    for p in rng.choice(np.arange(lo, hi), min(k, hi - lo), replace=False):
        s[p] = NT[(NT.index(s[p]) + int(rng.integers(1, 4))) % 4]
    return "".join(s)


def indel(rng, s, lo, hi):
    """One 1-3 nt insertion or deletion at a random position in [lo, hi)."""
    p, k = int(rng.integers(lo, hi)), int(rng.integers(1, 4))
    if rng.random() < 0.5:
        return s[:p] + "".join(NT[x] for x in rng.integers(0, 4, k)) + s[p:]
    return s[:p] + s[p + k:]


def homopolymer_edit(rng, s):
    """Lengthen or shorten the longest homopolymer run by one base (the commonest indel of real data)."""
    best, bp, i = 0, 0, 0
    while i < len(s):
        j = i
        while j < len(s) and s[j] == s[i]:
            j += 1
        if j - i > best:
            best, bp = j - i, i
        i = j
    return s[:bp] + s[bp] + s[bp:] if rng.random() < 0.5 else s[:bp] + s[bp + 1:]


# ---- mergePairs ----
def miseq_pairs(n, seed, rl=300, amp=(400, 481)):
    """2 x rl reads over amplicons of length in [amp[0], amp[1]): (pool, s1, s2, prefer) for merge_align, the reverse
    read already reverse-complemented.  A third of the reverse reads carry a substitution, an indel or a homopolymer edit inside the
    overlap; a few pairs do not overlap at all; some are truncated like truncLen = (280, 220)."""
    rng = np.random.default_rng(seed)
    pool, s1, s2 = [], [], []
    for it in range(n):
        a = rand_seq(rng, int(rng.integers(amp[0], amp[1])))
        f, r = a[:rl], a[-rl:]
        if it % 7 == 3:
            f, r = f[:280], r[-220:]
        ov = len(f) + len(r) - len(a)
        u = it % 6
        if ov > 20 and u == 1:
            r = substitute(rng, r, 1, 0, ov)
        elif ov > 20 and u == 3:
            r = indel(rng, r, 5, ov - 5)
        elif u == 5:
            r = homopolymer_edit(rng, r)
        if it % 17 == 11:
            r = rand_seq(rng, len(r))                                      # no overlap at all
        pool += [f, r]
        s1.append(len(pool) - 2)
        s2.append(len(pool) - 1)
    prefer = (1 + (np.arange(n) % 2)).astype(np.int32)
    return pool, np.asarray(s1, np.int32), np.asarray(s2, np.int32), prefer


def merge_batch_at(maxlen, n, seed, overlap=(20, 120), equal=False):
    """Pairs whose reads are at most `maxlen` long (one read exactly `maxlen`; all of them with `equal`), over amplicons
    that leave an overlap of overlap[0]..overlap[1] nt between equally long reads."""
    rng = np.random.default_rng(seed)
    pool, s1, s2 = [], [], []
    for it in range(n):
        rl = maxlen if it == 0 or equal else int(rng.integers(max(overlap[1] + 1, maxlen - 40), maxlen + 1))
        ov = int(rng.integers(overlap[0], min(overlap[1], rl) + 1))
        a = rand_seq(rng, 2 * rl - ov)
        f, r = a[:rl], a[-rl:]
        if it % 3 == 1:
            r = indel(rng, r, 2, ov - 2)
            if equal:                                                           # keep the length: pad or cut the far end
                r = (r + rand_seq(rng, 3))[:rl]
        elif it % 3 == 2:
            r = substitute(rng, r, 1, 0, ov)
        pool += [f, r[:maxlen]]
        s1.append(len(pool) - 2)
        s2.append(len(pool) - 1)
    assert max(len(x) for x in pool) == maxlen
    return pool, np.asarray(s1, np.int32), np.asarray(s2, np.int32), (1 + (np.arange(n) % 2)).astype(np.int32)


# ---- bimera ----
def bimera_pairs_at(maxlen, spread, nquery, seed, nsub=3):
    """(seqs, query, parent) for test_bimera_pairs: queries of length maxlen and parents of length maxlen - spread (so
    the batch spread is exactly `spread`); each query is followed by runs of two parents of the same length, which is
    what the 16-bit kernel pairs up.  Queries are two-parent bimeras (some one-off, some with an indel) of their
    parents or plain substitution variants; parents longer than the query occur too when spread > 0."""
    rng = np.random.default_rng(seed)
    lq, lp = maxlen, maxlen - spread
    seqs, q, p = [], [], []
    for it in range(nquery):
        root = rand_seq(rng, lq)
        a, b = substitute(rng, root, 8), substitute(rng, root, 12)
        bp = int(rng.integers(20, lq - 20))
        x = a[:bp] + b[bp:]
        if it % 3 == 1:
            x = substitute(rng, x, 1)
        elif it % 3 == 2:
            x = indel(rng, x, 10, lq - 10)
            x = (x + root)[:lq]
        k = len(seqs)
        seqs += [x, a[:lp], b[:lp], a[spread:], substitute(rng, root, 2)[:lp]]
        q += [k] * 4
        p += [k + 1, k + 2, k + 3, k + 4]
        if spread and it % 2:
            q += [k + 1, k + 2]                                              # parent-length queries against the long one
            p += [k, k]
    return seqs, np.asarray(q, np.int32), np.asarray(p, np.int32)


def bimera_table(nseq, nsample, seed, L, lenvar):
    from tools import synth
    seqs, mat = synth.bimera_table(nseq, nsample, L=L, seed=seed, lenvar=lenvar)
    mat[:, 1] = mat[:, 2] = np.maximum(mat[:, 1], mat[:, 2])                  # tied abundances
    return seqs, mat


def v34_table(nseq, nsample=8, seed=1):
    return bimera_table(nseq, nsample, seed, L=460, lenvar=60)


def pacbio_table(nseq, nsample=4, seed=1, L=1600, lenvar=200):
    return bimera_table(nseq, nsample, seed, L=L, lenvar=lenvar)


# ---- collapseNoMismatch ----
def collapse_table(nfam, seed, L=(400, 461), nsamp=6):
    """(mat, colnames): families of one ASV with truncated, end-shifted and prefix copies (nwhamming 0), SNP and indel
    neighbours (> 0) and homopolymer edits; duplicate columns and tied column sums."""
    rng = np.random.default_rng(seed)
    cols = []
    for _ in range(nfam):
        a = rand_seq(rng, int(rng.integers(L[0], L[1])))
        fam = [a, a[:-int(rng.integers(1, 30))], a[int(rng.integers(1, 30)):], substitute(rng, a, 1), indel(rng, a, 30, len(a) - 30),
               homopolymer_edit(rng, a), a[5:-5], "".join(NT[x] for x in rng.integers(0, 4, 7)) + a]
        cols += fam
    cols.append(cols[0])                                                        # a duplicate column
    mat = rng.integers(0, 50, (nsamp, len(cols))).astype(np.int32)
    mat[:, 3] = mat[:, 4]                                                       # tied column sums
    return mat, cols


def collapse_pairs_at(maxlen, n, seed, spread=30):
    """(seqs, query, ref): sequences of length maxlen - spread .. maxlen (one exactly maxlen) in pairs that are
    truncations, shifts, SNP or indel neighbours of each other."""
    rng = np.random.default_rng(seed)
    seqs, q, r = [], [], []
    half = spread // 2
    for it in range(n):
        a = rand_seq(rng, maxlen if it == 0 else int(rng.integers(maxlen - half, maxlen + 1)))
        u = it % 5
        b = [a[:-int(rng.integers(1, half))], a[int(rng.integers(1, half)):], substitute(rng, a, 1), indel(rng, a, 20, len(a) - 20),
             a][u]
        b = b[:maxlen]
        seqs += [a, b]
        q.append(len(seqs) - 1)
        r.append(len(seqs) - 2)
    assert max(len(s) for s in seqs) == maxlen and min(len(s) for s in seqs) >= maxlen - spread
    return seqs, np.asarray(q, np.int32), np.asarray(r, np.int32)


# ---- derep ----
def derep_reads(L, nvar, nreads, seed, qmax=41):
    """Reads of exactly L nt (plus proper prefixes of length L - 1 and L - 16 when L is long enough, which share key words
    with the full read), heavy duplication with tied abundances, qualities 0..qmax."""
    rng = np.random.default_rng(seed)
    base = [rand_seq(rng, L) for _ in range(nvar)]
    base += [b[:L - 1] for b in base[:2] if L > 1] + [b[:L - 16] for b in base[2:3] if L > 16]
    base += [base[0][:L - 1] + NT[(NT.index(base[0][-1]) + 1) % 4]]             # differs in the last base only
    reads = [base[k % len(base)] for k in range(2 * len(base))]                 # every unique twice: ties
    reads += [base[int(x)] for x in rng.integers(0, len(base), max(0, nreads - len(reads)))]
    perm = rng.permutation(len(reads))
    seqs = [reads[k] for k in perm]
    quals = [rng.integers(0, qmax + 1, len(s)).astype(np.uint8) for s in seqs]
    return seqs, quals


# ---- filterAndTrim ----
PACBIO_PRIMER = "AGGGTTTGATTATGGCTCAG"          # 27F (AGRGTTYGATYMTGGCTCAG) with its ambiguity codes resolved


def pacbio_reads(n, seed, primer=PACBIO_PRIMER, phix=None):
    """CCS-like reads, 1000-1700 nt: qualities mostly 60-93 with low stretches, a third reverse-complemented, some
    without the primer, some with an N or a long low-quality tail, some carrying a phiX fragment."""
    from tests.filter_ref import rc
    rng = np.random.default_rng(seed)
    reads = []
    for it in range(n):
        L = int(rng.integers(950, 1701))
        s = primer + rand_seq(rng, L - len(primer))
        q = np.clip(rng.normal(80, 12, L), 0, 93).astype(int)
        if it % 5 == 1:
            p = int(rng.integers(0, L - 50)); q[p:p + 50] = rng.integers(0, 15, 50)
        if it % 7 == 2:
            q[-int(rng.integers(100, 600)):] = rng.integers(0, 8, 1)[0]
        if it % 11 == 4:
            p = int(rng.integers(0, L)); s = s[:p] + "N" + s[p + 1:]
        if it % 13 == 5:
            s = rand_seq(rng, L)                                                # no primer on either strand
        if it % 9 == 6 and phix is not None:
            st = int(rng.integers(0, len(phix) - 200)); p = int(rng.integers(len(primer), L - 200))
            s = s[:p] + phix[st:st + 200] + s[p + 200:]
        if it % 17 == 8:
            q[:] = 93
        if it % 3 == 0:
            s, q = rc(s), q[::-1]
        reads.append((s, [int(x) for x in q]))
    return reads


def miseq_read_pairs(n, seed, rl=300):
    """2 x rl raw read pairs with Illumina-like qualities falling towards the 3' end, some low tails and Ns."""
    rng = np.random.default_rng(seed)
    out = []
    prof = np.clip(np.round(38 - 24 * (np.arange(rl) / (rl - 1)) ** 3), 2, 41)
    for it in range(n):
        mates = []
        for m in range(2):
            s = rand_seq(rng, rl)
            q = np.clip(np.round(prof + rng.normal(0, 4, rl)), 0, 41).astype(int)
            if (it + m) % 5 == 0:
                q[-int(rng.integers(10, 120)):] = int(rng.integers(0, 3))
            if (it + 3 * m) % 23 == 0:
                p = int(rng.integers(0, rl)); s = s[:p] + "N" + s[p + 1:]
            mates.append((s, [int(x) for x in q]))
        out.append(tuple(mates))
    return out

"""Plain restatement of the k-mer screen of one dada() round, in numpy with exact integers (test infrastructure).

For centre c and every raw r it restates raw_align's decision (/root/reference/src/nwalign_endsfree.cpp:44-56):
    kdist  = 1. - minsum / (min(len_c, len_r) - 5 + 1.)                      kmers.cpp:13-26 (uint16 dotsum)
    kodist = 1. - ordered / (min(len_c, len_r) - 5 + 1.), or -1 when gapless is off, and when SSE == 0 and the lengths differ
             (kord_dist, kmers.cpp:102-116; the SSE path kmers.cpp:121-150 compares min(len) - 4 positions whatever the lengths)
    kind   = 0 shrouded (kdist > cutoff), 1 gapless (band == 0 or kodist == kdist), 2 NW
with the greedy skip of cluster.cpp:127-131 in front (a skipped raw is not compared: kind 0, not counted).  5-mer counts are those
of assign_kmer (kmers.cpp:207-279, uint16 per 5-mer).  It also restates what the device's streaming tier derives from the same
counts: the presence bound, and whether a raw's repeated-5-mer list overflows (more than KREP distinct repeated 5-mers, or a count
above 64), so that tests can say which raws must reach k_classify.
"""
import numpy as np

K = 5
NK = 1 << (2 * K)
KREP = 48                      # dd_prescreen.cu: repeated-5-mer list entries per raw
REP_MAX = 64                   # largest count a list entry holds
_CODE = np.full(256, 255, np.uint8)
for _i, _c in enumerate(b"ACGT"):
    _CODE[_c] = _i


def encode(seq):
    a = _CODE[np.frombuffer(seq.encode("ascii"), np.uint8)]
    if (a == 255).any():
        raise ValueError("Unexpected nucleotide.")
    return a.astype(np.int64)


def kmers(seq):
    """5-mer index at every position 0 .. len - 5 (first base most significant, as assign_kmer)."""
    a = encode(seq)
    n = len(a) - K + 1
    km = np.zeros(n, np.int64)
    for j in range(K):
        km = km * 4 + a[j:j + n]
    return km


def kmer_counts(seq):
    return np.bincount(kmers(seq), minlength=NK).astype(np.uint16)


def kdist_of(ms, len1, len2):
    """kmers.cpp:23, float64 with the same operations."""
    return 1. - np.asarray(ms, np.float64) / ((np.minimum(len1, len2) - K).astype(np.float64) + 1.)


def _padded_kmers(seqs, idx):
    lens = np.array([len(seqs[i]) for i in idx], np.int64)
    W = int(lens.max()) - K + 1
    km = np.full((len(idx), W), NK, np.int64)                  # NK: padding, sorts behind every real 5-mer
    for row, i in enumerate(idx):
        k = kmers(seqs[i])
        km[row, :len(k)] = k
    return lens, km


def screen(seqs, centre, kdist_cutoff, reads=None, centre_reads=None, lock=None, greedy=False, use_kmers=True, gapless=True,
           band_size=16, SSE=2, rank=0, world=1, **_ignored):
    """-> dict of per-raw arrays (kind: -1 other rank / 0 / 1 / 2, minsum, ordered, kdist, kodist, bound, skipped, shrouded,
    overflow) and the round's counters align (raws compared) and shroud (raws shrouded)."""
    n = len(seqs)
    reads = np.zeros(n, np.int64) if reads is None else np.asarray(reads, np.int64)
    lock = np.zeros(n, bool) if lock is None else np.asarray(lock, bool)
    if centre_reads is None:
        centre_reads = int(reads[centre])
    owned = np.arange(n) % world == rank
    skipped = bool(greedy) & ((reads > centre_reads) | lock)
    cc = np.zeros(NK + 1, np.int64)
    cc[:NK] = kmer_counts(seqs[centre])
    ckm = kmers(seqs[centre])
    len1 = len(seqs[centre])
    ms = np.zeros(n, np.int64); om = np.zeros(n, np.int64); bound = np.zeros(n, np.int64); ovf = np.zeros(n, bool)
    lens = np.array([len(s) for s in seqs], np.int64)
    order = np.argsort(lens, kind="stable")                    # chunks of similar lengths: little padding
    lim = 1 << 22
    at = 0
    while at < n:
        m = 1
        while at + m < n and (m + 1) * int(lens[order[at + m]]) <= lim:
            m += 1
        idx = order[at:at + m]
        at += m
        l2, km = _padded_kmers(seqs, idx)
        W = km.shape[1]
        S = np.sort(km, axis=1)
        pos = np.arange(W)
        start = np.ones(S.shape, bool)
        start[:, 1:] = S[:, 1:] != S[:, :-1]
        first = np.maximum.accumulate(np.where(start, pos, 0), axis=1)
        occ = pos - first                                      # occurrence number of this 5-mer within the raw, from 0
        real = S < NK
        ms[idx] = (real & (occ < cc[S])).sum(1) & 0xFFFF        # sum_k min(c_raw[k], c_centre[k]), uint16 as the reference's dotsum
        distinct = (real & start).sum(1)
        shared = (real & start & (cc[S] > 0)).sum(1)
        bound[idx] = shared + (l2 - K + 1 - distinct)          # presence bound of dd_prescreen.cu
        run_len = np.zeros(S.shape, np.int64)                  # at the last entry of a run: its length
        end = np.ones(S.shape, bool)
        end[:, :-1] = S[:, 1:] != S[:, :-1]
        run_len[end] = (occ + 1)[end]
        nrep = (real & end & (run_len >= 2)).sum(1)
        ovf[idx] = (nrep > KREP) | (real & end & (run_len > REP_MAX)).any(1)
        ck = np.full(W, -1, np.int64)
        ck[:min(W, len(ckm))] = ckm[:W]
        nko = np.minimum(l2, len1) - K + 1
        om[idx] = ((km == ck[None, :]) & (pos[None, :] < nko[:, None])).sum(1) & 0xFFFF
    kdist = kdist_of(ms, len1, lens) if use_kmers else np.zeros(n)
    ko_valid = np.full(n, bool(use_kmers and gapless)) & ~((SSE == 0) & (lens != len1))
    kodist = np.where(ko_valid, kdist_of(om, len1, lens), -1.0)
    shrouded = np.asarray(use_kmers & (kdist > kdist_cutoff), bool)
    gl = (band_size == 0) | (bool(gapless) & (kodist == kdist))
    kind = np.where(shrouded, 0, np.where(gl, 1, 2))
    kind = np.where(skipped, 0, kind)
    kind = np.where(owned, kind, -1).astype(np.int32)
    act = owned & ~skipped
    return dict(kind=kind, minsum=ms, ordered=om, kdist=kdist, kodist=kodist, bound=bound, overflow=ovf, skipped=skipped,
                shrouded=shrouded & act, owned=owned, align=int(act.sum()), shroud=int((shrouded & act).sum()))

"""Numpy restatement of the classifier's contract (DESIGN.md 21) and the compiled reference's C-ABI.

Table in the stated float order, main and bootstrap sums as sequential fp32 sums (np.cumsum, never the pairwise
np.sum), the tie rule, the seeded draws with the reference's buffer layout, and the boot counts.  The sums take the
table as an argument, so the product's own table (fetched through its hook) can be fed in and the sums compared bit for
bit, while the table itself is compared with `table()` under the 1-ulp rule."""
import ctypes as C
import gzip
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
NK = 65536
NBOOT = 100
NA = -(2 ** 31)
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)
_CODE = np.full(256, -1, np.int64)
for _i, _c in enumerate(b"ACGT"):
    _CODE[_c] = _i


def mix(z):
    """splitmix64 finaliser on uint64 arrays (wrapping arithmetic)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _add(a, b):
    with np.errstate(over="ignore"):
        return np.asarray(a, np.uint64) + np.asarray(b, np.uint64)


def kmer_windows(seq):
    """-> int64 [len - 7]: the 8-mer at each window, -1 where a letter is not A/C/G/T."""
    b = np.frombuffer(seq.encode() if isinstance(seq, str) else seq, np.uint8)
    if len(b) < 8:
        return np.zeros(0, np.int64)
    c = _CODE[b]
    W = len(b) - 7
    km = np.zeros(W, np.int64)
    bad = np.zeros(W, bool)
    for t in range(8):
        km = km * 4 + np.maximum(c[t:t + W], 0)
        bad |= c[t:t + W] < 0
    km[bad] = -1
    return km


def karray(seq):
    w = kmer_windows(seq)
    return np.sort(w[w >= 0])


def rc_kmers(k):
    k = np.asarray(k, np.int64)
    c = (~k) & 0xFFFF
    r = np.zeros_like(k)
    for _ in range(8):
        r = (r << 2) | (c & 3)
        c >>= 2
    return r


def table(refs, ref_to_genus, ngenus):
    """float32 [ngenus, 65536]: (float)log((double)(((float)cnt + prior) / (float)(M_g + 1)))."""
    nref = len(refs)
    pres = []
    ck = np.zeros(NK, np.int64)
    cnt = np.zeros((ngenus, NK), np.float32)
    for r, g in zip(refs, ref_to_genus):
        k = np.unique(kmer_windows(r))
        k = k[k >= 0]
        ck[k] += 1
        cnt[g - 1, k] += np.float32(1)
        pres.append(k)
    prior = ((ck.astype(np.float64) + 0.5) / (1.0 + nref)).astype(np.float32)
    gnp1 = np.zeros(ngenus, np.float32)
    for g in ref_to_genus:
        gnp1[g - 1] += np.float32(1)
    gnp1 += np.float32(1)
    x = (cnt + prior[None, :]) / gnp1[:, None]                  # float32 add, float32 divide
    return np.log(x.astype(np.float64)).astype(np.float32)


def seq_sums(lgk, arrays):
    """Sequential fp32 sums: lgk [G, 65536], arrays [R, n] of k-mers -> float32 [R, G]."""
    arrays = np.asarray(arrays, np.int64)
    if arrays.shape[1] == 0:
        return np.zeros((arrays.shape[0], lgk.shape[0]), np.float32)
    out = np.empty((arrays.shape[0], lgk.shape[0]), np.float32)
    for r in range(arrays.shape[0]):
        out[r] = np.cumsum(lgk[:, arrays[r]], axis=1, dtype=np.float32)[:, -1]
    return out


def tie_pick(lp, seed, j, r):
    """The tie rule over float32 lp [G] -> (genus 0-based, tie set size, gap to the best other genus)."""
    m = lp.max()
    tie = np.flatnonzero(lp == m)
    g = int(tie[0])
    if len(tie) > 1:
        jb = mix(_add(mix(np.uint64(seed)), np.uint64(j)))
        h = mix(_add(jb, (np.uint64(r) << np.uint64(32)) | tie.astype(np.uint64)))
        g = int(tie[np.lexsort((tie, h))[0]])
    rest = lp[lp != m]
    gap = float(m) - float(rest.max()) if rest.size else np.inf
    return g, len(tie), gap


def draws(seed, n0, count):
    """Seeded uniforms n0 .. n0 + count - 1 of the virtual buffer."""
    sb = mix(np.uint64(seed) ^ np.uint64(0x9E3779B97F4A7C15))
    n = np.arange(count, dtype=np.uint64) + np.uint64(n0)
    return (mix(_add(sb, n)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def max_arraylen(seqs):
    return max([len(s) - 7 for s in seqs if len(s) >= 7] or [0])


def unifs_buffer(seqs, seed):
    """The full buffer the reference's runif would return, filled with the seeded draws."""
    return draws(seed, 0, len(seqs) * NBOOT * (max_arraylen(seqs) // 8))


def classify(lgk, genusmat, seqs, try_rc, seed, unifs=None, only=None):
    """-> dict(tax, boot, boot_tax, logp, used_rc, strict [nseq] main arg-max strict, boot_strict [nseq, 100],
    gap / boot_gap margins to the runner-up).  only: restate just these query indices (the others stay NA)."""
    n = len(seqs)
    nl = genusmat.shape[1]
    mal = max_arraylen(seqs)
    R = {"tax": np.full(n, NA, np.int32), "boot": np.zeros((n, nl), np.int32), "boot_tax": np.full((n, NBOOT), NA, np.int32),
         "logp": np.full(n, np.nan, np.float32), "used_rc": np.zeros(n, bool), "strict": np.ones(n, bool),
         "boot_strict": np.ones((n, NBOOT), bool), "gap": np.full(n, np.inf), "boot_gap": np.full((n, NBOOT), np.inf)}
    for j in (range(n) if only is None else only):
        s = seqs[j]
        if len(s) < 50:
            continue
        ka = karray(s)
        L = len(ka)
        if L > 9999:
            raise ValueError("query over 9999 k-mers")
        lp = seq_sums(lgk, ka[None, :])[0]
        g, nt, gap = tie_pick(lp, seed, j, 100)
        best, strict = lp[g], nt == 1
        if try_rc:
            kr = np.sort(rc_kmers(ka))
            lpr = seq_sums(lgk, kr[None, :])[0]
            gr, ntr, gapr = tie_pick(lpr, seed, j, 101)
            ogap = abs(float(lpr.max()) - float(lp.max()))        # the orientation is decided by a margin too
            if lpr[gr] > best:
                ka, g, best, nt, gap = kr, gr, lpr[gr], ntr, gapr
                R["used_rc"][j] = True
            strict, gap = nt == 1 and ogap > 0, min(gap, ogap)
        R["tax"][j], R["logp"][j], R["strict"][j], R["gap"][j] = g + 1, best, strict, gap
        n8 = L // 8
        u = unifs[j * mal: j * mal + NBOOT * n8] if unifs is not None else draws(seed, j * mal, NBOOT * n8)
        pos = np.minimum((L * u).astype(np.int64), max(L - 1, 0))
        barr = ka[pos].reshape(NBOOT, n8) if n8 else np.zeros((NBOOT, 0), np.int64)
        bl = seq_sums(lgk, barr)
        for b in range(NBOOT):
            bg, bnt, bgap = tie_pick(bl[b], seed, j, b)
            R["boot_tax"][j, b] = bg + 1
            R["boot_strict"][j, b] = bnt == 1
            R["boot_gap"][j, b] = bgap
            for lev in range(nl):
                if genusmat[bg, lev] != genusmat[g, lev]:
                    break
                R["boot"][j, lev] += 1
    return R


# ---- fixtures ----
def read_fasta(path):
    op = gzip.open if path.endswith(".gz") else open
    ids, seqs = [], []
    with op(path, "rt") as f:
        for line in f:
            line = line.rstrip("\r\n")
            if line.startswith(">"):
                ids.append(line[1:])
                seqs.append([])
            elif ids:
                seqs[-1].append(line.strip())
    return ids, ["".join(s).upper() for s in seqs]


def ten16s():
    """ten_16s.100.fa.gz with its `tax=d:..,g:..;` headers converted to DADA2's `Bacteria;...;Genus;` form."""
    ids, seqs = read_fasta(os.path.join(GOLDEN, "ten_16s.100.fa.gz"))
    out = []
    for h in ids:
        t = h.split("tax=", 1)[1].rstrip(";")
        out.append(";".join(f.split(":", 1)[1] for f in t.split(",")) + ";")
    return out, seqs


def revcomp(s):
    return s.translate(str.maketrans("ACGTN", "TGCAN"))[::-1]


# ---- the compiled reference (oracle/_ref/libdada2ref_taxonomy.so, built by oracle/taxonomy.mk) ----
_REF = None


def ref_lib():
    global _REF
    if _REF is None:
        p = os.path.join(ROOT, "oracle", "_ref", "libdada2ref_taxonomy.so")
        if not os.path.exists(p):
            return None
        _REF = C.CDLL(p)
        _REF.ref_assign_taxonomy.argtypes = [C.c_int, C.c_char_p, C.c_void_p, C.c_char_p, C.c_void_p, C.c_int, C.c_char_p, C.c_void_p,
                                             C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_int,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    return _REF


def _cat(seqs):
    b = [s.encode() for s in seqs]
    off = np.zeros(len(b) + 1, np.int64)
    np.cumsum([len(x) for x in b], out=off[1:])
    return b"".join(b) or b"\0", off


def ref_assign(seqs, refs, ref_to_genus, genusmat, try_rc, unifs, nthreads=1):
    """C_assign_taxonomy2 of the reference with injected uniforms -> dict(tax, boot, boot_tax)."""
    L = ref_lib()
    n, nl = len(seqs), genusmat.shape[1]
    sc, so = _cat(seqs)
    rcc, rco = _cat([revcomp(s) for s in seqs])
    fc, fo = _cat(refs)
    rg = np.ascontiguousarray(ref_to_genus, np.int32)
    gm = np.ascontiguousarray(genusmat, np.int32)
    u = np.ascontiguousarray(unifs, np.float64)
    tax = np.zeros(n, np.int32)
    boot = np.zeros((n, nl), np.int32)
    bt = np.zeros((n, NBOOT), np.int32)
    err = C.create_string_buffer(512)
    if L.ref_assign_taxonomy(n, sc, so.ctypes.data, rcc, rco.ctypes.data, len(refs), fc, fo.ctypes.data, rg.ctypes.data, gm.shape[0], nl,
                             gm.ctypes.data, int(bool(try_rc)), u.ctypes.data, u.size, int(nthreads), tax.ctypes.data, boot.ctypes.data,
                             bt.ctypes.data, err, 512):
        raise RuntimeError(err.value.decode())
    return {"tax": tax, "boot": boot, "boot_tax": bt}

"""mergePairs cases shared by the CPU, emulator and GPU tests: small hand-built samples and a synthetic multi-sample set.

A dada result here carries what mergePairs reads: `map` (unique -> cluster, NA = INT32_MIN) and `clustering` (sequence, n0,
abundance, birth_ham); a derep result carries `uniques` and `map` (read -> unique)."""
import numpy as np

from tests.paired_ref import NA, rc

AMP = ("GTATCGGCTACCGCAAAAATAGTACCCTATTTACGCGGGATGTCCTAACGATCAGTTTCATGTAAGCCTAGCCTACAACGGCATTAACATGGCGTATACTTATTCC")


def sub(s, i):
    return s[:i] + "ACGT"[("ACGT".index(s[i]) + 1) % 4] + s[i + 1:]


def dada_obj(seqs, n0, dmap, rc_seqs=False):
    seqs = [rc(s) for s in seqs] if rc_seqs else list(seqs)
    return {"clustering": {"sequence": seqs, "n0": np.asarray(n0, np.int32), "abundance": np.asarray(n0, np.int32) + 1,
                           "birth_ham": np.arange(len(seqs), dtype=np.int32)},
            "map": np.asarray([NA if x is None else x for x in dmap], np.int32)}


def derep_obj(nuniq, rmap):
    return {"uniques": ["A"] * nuniq, "map": np.asarray([NA if x is None else x for x in rmap], np.int32)}


def hand_sample():
    """Two forward clusters (F2 carries a substitution outside the overlap), two reverse clusters (R2 carries one inside the
    overlap), an uncorrected forward unique (NA in dadaF$map), an NA read in derepF$map, and an abundance tie."""
    F = [AMP[:60], sub(AMP[:60], 5)]
    R = [AMP[40:], sub(AMP, 50)[40:]]
    dF = dada_obj(F, [5, 1], [1, 2, 1, None])
    dR = dada_obj(R, [2, 9], [1, 2, 1], rc_seqs=True)
    rF = derep_obj(4, [1, 2, 1, 4, 3, None, 2, 1, 2])
    rR = derep_obj(3, [1, 1, 2, 1, 3, 1, 1, 2, 1])
    return dF, rF, dR, rR


def empty_sample():
    """Every read has an NA on one side: no pairing."""
    dF = dada_obj([AMP[:60]], [3], [1, None])
    dR = dada_obj([AMP[40:]], [3], [None, 1], rc_seqs=True)
    return dF, derep_obj(2, [1, 2, 2]), dR, derep_obj(2, [1, 2, 1])


def overhang_sample():
    """The reverse read runs past the forward read's start (amplicon shorter than the reads): trimOverhang trims it."""
    F = [AMP[10:80]]
    R = [AMP[0:70], sub(AMP[0:70], 40)]
    dF = dada_obj(F, [4], [1, 1])
    dR = dada_obj(R, [4, 5], [1, 2], rc_seqs=True)
    return dF, derep_obj(2, [1, 2, 1, 1]), dR, derep_obj(2, [1, 1, 2, 2])


def synth_set(nsamples, nreads, seed, namp=12, lenlo=253, lenhi=480, readlen=250, na_frac=0.01):
    """nsamples samples of 2 x readlen reads over namp amplicons of lenlo..lenhi nt; some amplicons have a variant with a
    substitution or an indel in the overlap on the reverse side.  Cluster sets and orders differ per sample, the dada maps
    have uncorrected (NA) uniques and the derep maps NA reads."""
    rng = np.random.default_rng(seed)
    amps = ["".join("ACGT"[i] for i in rng.integers(0, 4, int(rng.integers(lenlo, lenhi + 1)))) for _ in range(namp)]
    Fall = [a[:readlen] for a in amps]
    Rall = [a[-readlen:] for a in amps]
    for a in list(amps[:namp // 3]):
        r = a[-readlen:]
        ov = 2 * readlen - len(a)                                  # overlap length; the overlap is r[:ov]
        p = int(rng.integers(0, max(ov, 1)))
        Rall.append(sub(r, p) if rng.random() < 0.5 else r[:p] + r[p + 1:] + "A")
    var = {k: namp + k for k in range(namp // 3)}                   # amplicon -> its variant's index in Rall
    out = []
    for s in range(nsamples):
        kF = rng.permutation(namp)[:int(rng.integers(3, namp + 1))]
        extra = [var[k] for k in kF if k in var] + [int(k) for k in rng.permutation(namp)[:2]]
        F = [Fall[k] for k in kF]
        R = [Rall[k] for k in kF] + [Rall[k] for k in extra]        # cluster c < len(F): the true partner of forward cluster c
        nF, nR = len(F), len(R)
        nuF, nuR = nF * 3, nR * 3
        dmF = [(u % nF) + 1 for u in range(nuF)]
        dmR = [(u % nR) + 1 for u in range(nuR)]
        for u in range(nF, nuF):
            if rng.random() < 0.2:
                dmF[u] = None
        for u in range(nR, nuR):
            if rng.random() < 0.2:
                dmR[u] = None
        n = nreads
        w = rng.dirichlet(np.ones(nuF) * 0.5)
        mF = rng.choice(nuF, size=n, p=w) + 1
        c = (mF - 1) % nF                                          # the read's forward cluster (when not NA)
        vpos = {k: nF + i for i, k in enumerate(e for e in extra[:len(extra) - 2])}
        vc = np.array([vpos.get(var.get(int(k), -1), -1) for k in kF])[c]
        cR = np.where((vc >= 0) & (rng.random(n) < 0.3), vc, c)     # some reads carry the variant reverse read
        cR = np.where(rng.random(n) < 0.1, rng.integers(0, nR, n), cR)  # and some a wrong partner
        mR = cR + nR * rng.integers(0, 3, n) + 1
        mF[:nuF], mR[:nuR] = np.arange(1, nuF + 1), np.arange(1, nuR + 1)      # every unique occurs
        mF = mF.astype(np.int32); mR = mR.astype(np.int32)
        mF[nuF:][rng.random(n - nuF) < na_frac] = NA
        mR[nuR:][rng.random(n - nuR) < na_frac] = NA
        n0F = rng.integers(1, 1000, nF)
        n0R = rng.integers(1, 1000, nR)
        out.append((dada_obj(F, n0F, dmF), derep_obj(nuF, mF), dada_obj(R, n0R, dmR, rc_seqs=True), derep_obj(nuR, mR)))
    return out

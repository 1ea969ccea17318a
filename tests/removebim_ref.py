"""Test reference for removeBimeraDenovo: the R loops of isBimeraDenovo (R/chimeras.R:105-150) and removeBimeraDenovo
(:294-346) restated over the oracle's C_is_bimera / C_table_bimera2.  The backend is `oracle.ref` (the reference's
chimera.cpp, compiled unmodified) when oracle/_ref holds it and `oracle.port` (the CPU restatement) otherwise; both can be
pinned by name.  Sequence tables are (mat [nrow, ncol], colnames)."""
import numpy as np

DEFAULTS = dict(minFoldParentOverAbundance=2, minParentAbundance=8, allowOneOff=False, minOneOffParentDistance=4, maxShift=16)
TABLE_DEFAULTS = dict(minSampleFraction=0.9, ignoreNNegatives=1, minFoldParentOverAbundance=1.5, minParentAbundance=2, allowOneOff=False,
                      minOneOffParentDistance=4, maxShift=16)


def backend(name=None):
    from oracle import port, ref
    if name == "port" or (name is None and not ref.available()):
        return port
    return ref


def is_bimera_denovo(seqs, abunds, queries=None, backend_name=None, **rule):
    """isBimeraDenovo on one uniques vector whose names may repeat: getUniques sums duplicates (tapply), loopFun runs on
    every collapsed sequence, and the verdicts go back to the entries with %in%.  queries: optional bool per entry; an
    unset entry is not evaluated (FALSE unless a copy of it is).  -> bool per entry."""
    r = dict(DEFAULTS)
    r.update(rule)
    B = backend(backend_name)
    tot, ask = {}, {}
    for n, (s, a) in enumerate(zip(seqs, abunds)):
        tot[s] = tot.get(s, 0) + int(a)
        ask[s] = ask.get(s, False) or queries is None or bool(queries[n])
    useqs = list(tot)
    ab = [tot[s] for s in useqs]
    bims = set()
    for i, sq in enumerate(useqs):                                                      # loopFun, :124-133
        if not ask[sq]:
            continue
        pars = [useqs[k] for k in range(len(useqs)) if ab[k] > r["minFoldParentOverAbundance"] * ab[i] and ab[k] > r["minParentAbundance"]]
        if len(pars) >= 2 and B.is_bimera(sq, pars, allow_one_off=bool(r["allowOneOff"]), min_one_off_par_dist=int(r["minOneOffParentDistance"]),
                                          max_shift=int(r["maxShift"])):
            bims.add(sq)
    return np.array([s in bims for s in seqs], bool)                                    # seqs.input %in% seqs[bims], :150


def denovo_flags(mat, seqs, zero_queries, device=0, backend_name=None, **rule):
    """The contract of dada2_b200.bimera.denovo_flags (distinct seqs), restated: isBimeraDenovo on every row; with
    zero_queries unset a zero cell is not a query."""
    mat = np.asarray(mat)
    return np.array([is_bimera_denovo(seqs, row, None if zero_queries else row > 0, backend_name, **rule) for row in mat],
                    bool).reshape(mat.shape)


def per_sample_flags(mat, seqs, backend_name=None, **rule):
    """t(apply(seqtab, 1, isBimeraDenovo)) (R/chimeras.R:325): every cell evaluated, zero counts included."""
    mat = np.asarray(mat)
    return np.array([is_bimera_denovo(seqs, row, None, backend_name, **rule) for row in mat], bool).reshape(mat.shape)


def pooled_flags(mat, seqs, backend_name=None, **rule):
    """isBimeraDenovo(seqtab) (:321): getUniques(matrix) = as.integer(colSums(seqtab))."""
    return is_bimera_denovo(seqs, np.asarray(mat).sum(axis=0, dtype=np.int64), None, backend_name, **rule)


def consensus_flags(mat, seqs, backend_name=None, **kw):
    """isBimeraDenovoTable (:220-250) over C_table_bimera2."""
    o = dict(TABLE_DEFAULTS)
    o.update(kw)
    nflag, nsam = backend(backend_name).table_bimera(mat, list(seqs), min_fold=o["minFoldParentOverAbundance"], min_abund=o["minParentAbundance"],
                                                     allow_one_off=bool(o["allowOneOff"]), min_one_off_par_dist=o["minOneOffParentDistance"],
                                                     max_shift=o["maxShift"])
    nflag, nsam = nflag.astype(np.int64), nsam.astype(np.int64)
    return (nflag >= nsam) | ((nflag > 0) & (nflag >= (nsam - o["ignoreNNegatives"]) * o["minSampleFraction"]))


def remove_table(mat, cols, method="consensus", flags=None, backend_name=None, **kw):
    """removeBimeraDenovo's matrix branch (:319-337) -> (mat, cols).  flags: the method's flags when already known
    (per-sample: the full cell matrix)."""
    mat = np.asarray(mat)
    if method == "per-sample":
        bim = per_sample_flags(mat, cols, backend_name, **kw) if flags is None else np.asarray(flags, bool)
        out = mat.copy()
        out[bim] = 0
        keep = out.sum(axis=0, dtype=np.int64) != 0
        return out[:, keep], [c for c, k in zip(cols, keep) if k]
    if flags is not None:
        bim = np.asarray(flags, bool)
    elif method == "pooled":
        bim = pooled_flags(mat, cols, backend_name, **kw)
    else:
        bim = consensus_flags(mat, cols, backend_name, **kw)
    return mat[:, ~bim], [c for c, b in zip(cols, bim) if not b]

"""Sequence tables: makeSequenceTable and collapseNoMismatch (R/multiSample.R:31-55, :104-160), plus nwhamming
(R/misc.R:216-220) batched over pairs.

collapseNoMismatch's double loop over the table's columns (:125-144) runs in libdada2b.so behind
include/dada2b_collapse.h: the prefix screen, the exact overlap filter and the alignments on the GPU, the greedy order on
the host.  This module restates the R around it (duplicate columns, query order, output columns and their order) and only
marshals.  No CPU fallback.

A table is (mat, colnames, rownames): mat is an int32 [nsample, nseq] matrix like R's seqtab (rows = samples).
"""
import ctypes as C
import sys

import numpy as np

from . import api
from .bimera import _pack_seqs

ERRLEN = 256


class CollapseOpts(C.Structure):
    _fields_ = [("min_overlap", C.c_int32), ("match", C.c_int32), ("mismatch", C.c_int32), ("gap_p", C.c_int32), ("band", C.c_int32),
                ("vec", C.c_int32)]


class CollapseStats(C.Structure):
    _fields_ = [("n_candidates", C.c_int64), ("n_filtered", C.c_int64), ("n_aligned", C.c_int64), ("n_zero", C.c_int64),
                ("n_cells", C.c_int64), ("n_blocks", C.c_int64), ("gpu_launches", C.c_int64), ("ms_device", C.c_double),
                ("ms_k_align", C.c_double), ("ms_total", C.c_double)]


_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_collapse_default_opts.argtypes = [P(CollapseOpts)]
        L.dada2b_collapse_nomismatch.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, P(CollapseOpts), C.c_int32, C.c_void_p,
                                                 P(CollapseStats), C.c_char_p]
        L.dada2b_test_collapse_pairs.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                                 P(CollapseOpts), C.c_int32, C.c_void_p, C.c_char_p]
        _BOUND = True
    return L


def _opts(minOverlap, match, mismatch, gap, band, vec):
    return CollapseOpts(int(minOverlap), int(match), int(mismatch), int(gap), int(band), int(bool(vec)))


def collapse_reps(seqs, minOverlap=20, vec=True, band=-1, match=5, mismatch=-4, gap=-8, device=0, return_stats=False):
    """The loop of R/multiSample.R:125-144 over distinct sequences given in query order.  -> int32 rep[nseq]: the position
    of the sequence that seqs[j] collapses into, or j where seqs[j] is kept."""
    buf, off = _pack_seqs(seqs)
    rep = np.zeros(len(seqs), np.int32)
    st = CollapseStats()
    eb = C.create_string_buffer(ERRLEN)
    o = _opts(minOverlap, match, mismatch, gap, band, vec)
    rc = _lib().dada2b_collapse_nomismatch(len(seqs), buf, off.ctypes.data, C.byref(o), int(device), rep.ctypes.data, C.byref(st), eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    if return_stats:
        return rep, {k: getattr(st, k) for k, _ in CollapseStats._fields_}
    return rep


def test_collapse_pairs(seqs, query, ref, minOverlap=20, vec=True, band=-1, match=5, mismatch=-4, gap=-8, device=0):
    """Stage hook: -> int32[npairs, 3] = (prefix screen passes, overlap filter sends the pair to alignment,
    nwhamming(seqs[query[x]], seqs[ref[x]])); the last is always aligned on the device."""
    buf, off = _pack_seqs(seqs)
    q = np.ascontiguousarray(query, dtype=np.int32)
    r = np.ascontiguousarray(ref, dtype=np.int32)
    if len(q) != len(r):
        raise api.Dada2bError("dada2b: query and ref must have the same length.")
    out = np.zeros((max(len(q), 1), 3), np.int32)
    eb = C.create_string_buffer(ERRLEN)
    o = _opts(minOverlap, match, mismatch, gap, band, vec)
    rc = _lib().dada2b_test_collapse_pairs(len(seqs), buf, off.ctypes.data, len(q), q.ctypes.data, r.ctypes.data, C.byref(o), int(device),
                                           out.ctypes.data, eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    return out[:len(q)]


test_collapse_pairs.__test__ = False


def nwhamming(s1, s2, vec=False, band=-1, match=5, mismatch=-4, gap=-8, device=0):
    """R/misc.R:216-220 (nwalign, then C_eval_pair's mismatch + indel), vectorised over pairs like R's Vectorize:
    strings or equal-length lists of strings.  -> int, or int32 array for lists."""
    one = isinstance(s1, str) and isinstance(s2, str)
    a = [s1] if isinstance(s1, str) else list(s1)
    b = [s2] if isinstance(s2, str) else list(s2)
    if len(a) == 1 and len(b) > 1:
        a = a * len(b)
    if len(b) == 1 and len(a) > 1:
        b = b * len(a)
    if len(a) != len(b):
        raise api.Dada2bError("dada2b: nwhamming needs pairs of sequences.")
    out = test_collapse_pairs(a + b, np.arange(len(a)), np.arange(len(a), 2 * len(a)), minOverlap=0, vec=vec, band=band, match=match,
                              mismatch=mismatch, gap=gap, device=device)[:, 2]
    return int(out[0]) if one else out


def _order_desc(v):
    """R's order(v, decreasing=TRUE) for integer keys: radix sort, stable (ties keep column order)."""
    return np.argsort(-np.asarray(v, dtype=np.int64), kind="stable")


def _order_cols(mat, cols, orderBy):
    if orderBy is None:
        return mat, cols
    if orderBy == "abundance":
        o = _order_desc(mat.sum(axis=0, dtype=np.int64))
    elif orderBy == "nsamples":
        o = _order_desc((mat > 0).sum(axis=0))
    else:
        return mat, cols
    return mat[:, o], [cols[k] for k in o]


def _colsums(mat):
    cs = mat.sum(axis=0, dtype=np.int64)
    if len(cs) and cs.max() > np.iinfo(np.int32).max:
        raise api.Dada2bError("dada2b: a column sum exceeds the int32 range (R would return NA).")
    return cs


def _is_merger(s):
    return isinstance(s, dict) and "clustering" not in s and isinstance(s.get("sequence"), (list, tuple)) and "abundance" in s


def _merger_uniques(m):
    """getUniques' data.frame branch (R/misc.R:42-60): abundance by sequence; duplicated sequences (e.g. the "" of rejected
    rows kept by returnRejects) are summed with tapply, which sorts the names."""
    seqs, ab = list(m["sequence"]), [int(a) for a in m["abundance"]]
    if len(set(seqs)) == len(seqs):
        return dict(zip(seqs, ab))
    print("Duplicate sequences detected and merged.", file=sys.stderr)
    tot = {}
    for sq, a in zip(seqs, ab):
        tot[sq] = tot.get(sq, 0) + a
    return {sq: tot[sq] for sq in sorted(tot)}


def makeSequenceTable(samples, orderBy="abundance"):
    """R/multiSample.R:31-55.  samples: a list of samples, or a dict name -> sample; a sample is a {sequence: count} map,
    a dada_uniques result (its clustering's sequence / abundance) or a mergePairs merger (its sequence / abundance).
    -> (int32 mat [nsample, nseq], colnames, rownames)"""
    if _is_merger(samples) or (isinstance(samples, dict) and not all(isinstance(v, (dict, list, tuple)) for v in samples.values())):
        samples = [samples]
    names = list(samples.keys()) if isinstance(samples, dict) else None
    vals = list(samples.values()) if isinstance(samples, dict) else list(samples)
    unqs = []
    for s in vals:
        if isinstance(s, dict) and "clustering" in s:                      # getUniques(dada) = clustering's abundance by sequence
            cl = s["clustering"]
            s = dict(zip(cl["sequence"], (int(a) for a in cl["abundance"])))
        elif _is_merger(s):
            s = _merger_uniques(s)
        unqs.append(dict(s))
    cols, index = [], {}
    for u in unqs:
        for sq in u:
            if sq not in index:
                index[sq] = len(cols)
                cols.append(sq)
    mat = np.zeros((len(unqs), len(cols)), np.int32)
    for i, u in enumerate(unqs):
        for sq, n in u.items():
            mat[i, index[sq]] = n
    mat, cols = _order_cols(mat, cols, orderBy)
    return mat, cols, names


def collapseNoMismatch(seqtab, colnames, minOverlap=20, orderBy="abundance", identicalOnly=False, vec=True, band=-1, match=5, mismatch=-4,
                       gap=-8, rownames=None, device=0, return_stats=False):
    """R/multiSample.R:104-160.  seqtab: int [nsample, ncol] with sequences `colnames` (duplicates allowed).
    -> (int32 mat, colnames), or (mat, colnames, stats) with return_stats (stats is None when nothing was aligned)."""
    mat = np.asarray(seqtab)
    if mat.ndim != 2 or mat.shape[1] != len(colnames):
        raise api.Dada2bError("Input must be a valid sequence table.")
    mat = mat.astype(np.int64)
    cols = list(colnames)
    # :106-114 duplicate columns are added into the first column of that name
    first = {}
    keep = []
    for k, sq in enumerate(cols):
        if sq in first:
            mat[:, first[sq]] += mat[:, k]
        else:
            first[sq] = k
            keep.append(k)
    mat = mat[:, keep]
    cols = [cols[k] for k in keep]
    if mat.size and np.abs(mat).max() > np.iinfo(np.int32).max:
        raise api.Dada2bError("dada2b: a table entry exceeds the int32 range (R would return NA).")
    mat = mat.astype(np.int32)
    stats = None
    if identicalOnly or not cols:
        return (mat, cols, stats) if return_stats else (mat, cols)
    # :118-119 queries in decreasing column sum, ties in column order
    qord = _order_desc(_colsums(mat))
    seqs = [cols[k] for k in qord]
    rep = collapse_reps(seqs, minOverlap, vec, band, match, mismatch, gap, device, return_stats)
    if return_stats:
        rep, stats = rep
    # :120-144 collapsed counts go into the representative's column
    collapsed = np.zeros(mat.shape, np.int64)
    for j, k in enumerate(qord):
        collapsed[:, qord[rep[j]]] += mat[:, k]
    kept = np.zeros(len(cols), bool)
    kept[qord[rep == np.arange(len(seqs))]] = True
    out = collapsed[:, kept]
    ocols = [c for c, k in zip(cols, kept) if k]
    if len(ocols) and out.sum(axis=0).max() > np.iinfo(np.int32).max:
        raise api.Dada2bError("dada2b: a column sum exceeds the int32 range (R would return NA).")
    out = out.astype(np.int32)
    # :147-156 orderBy, then column sums again whatever orderBy was
    out, ocols = _order_cols(out, ocols, orderBy)
    out, ocols = _order_cols(out, ocols, "abundance")
    return (out, ocols, stats) if return_stats else (out, ocols)

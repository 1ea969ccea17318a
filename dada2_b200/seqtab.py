"""Sequence tables: makeSequenceTable, collapseNoMismatch and mergeSequenceTables (R/multiSample.R:31-55, :104-160,
:290-364), plus nwhamming (R/misc.R:216-220) batched over pairs on the public aligner (align.py).

collapseNoMismatch's double loop over the table's columns (:125-144) runs in libdada2b.so behind
include/dada2b_collapse.h: the prefix screen, the exact overlap filter and the alignments on the GPU, the greedy order on
the host.  This module restates the R around it (duplicate columns, query order, output columns and their order) and only
marshals.  mergeSequenceTables validates and names the samples here; everything about its columns (the union, tryRC's
re-orientation, the accumulation and the order) is one call behind include/dada2b_seqtab.h.  No CPU fallback.

A table is (mat, colnames, rownames): mat is an int32 [nsample, nseq] matrix like R's seqtab (rows = samples).
"""
import ctypes as C
import os
import sys
import warnings

import numpy as np

from . import align, api
from .bimera import _pack_seqs

ERRLEN = 256


class CollapseOpts(C.Structure):
    _fields_ = [("min_overlap", C.c_int32), ("match", C.c_int32), ("mismatch", C.c_int32), ("gap_p", C.c_int32), ("band", C.c_int32),
                ("vec", C.c_int32)]


class CollapseStats(C.Structure):
    _fields_ = [("n_candidates", C.c_int64), ("n_filtered", C.c_int64), ("n_aligned", C.c_int64), ("n_zero", C.c_int64),
                ("n_cells", C.c_int64), ("n_blocks", C.c_int64), ("gpu_launches", C.c_int64), ("ms_device", C.c_double),
                ("ms_k_align", C.c_double), ("ms_total", C.c_double)]


class SeqtabMergeIn(C.Structure):
    _fields_ = [("ntab", C.c_int32), ("nrow", C.c_void_p), ("ncol", C.c_void_p), ("names", C.c_char_p), ("name_off", C.c_void_p),
                ("row_out", C.c_void_p), ("entries", C.c_void_p), ("nrow_out", C.c_int32), ("try_rc", C.c_int32), ("order_by", C.c_int32)]


class SeqtabMergeOut(C.Structure):
    _fields_ = [("ncol_out", C.c_int32), ("name_src", C.POINTER(C.c_int32)), ("mat", C.POINTER(C.c_int32)), ("n_rc", C.c_int64),
                ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("ms_h2d", C.c_double),
                ("ms_kernels", C.c_double), ("ms_d2h", C.c_double), ("ms_device", C.c_double), ("ms_total", C.c_double)]


MERGE_STATS = ("n_rc", "gpu_launches", "h2d_bytes", "d2h_bytes", "ms_h2d", "ms_kernels", "ms_d2h", "ms_device", "ms_total")
ORDER_BY = {"abundance": 1, "nsamples": 2}        # DADA2B_ORDER_*; None and any other string: 0, the first-seen order

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
        L.dada2b_merge_seqtabs.argtypes = [P(SeqtabMergeIn), C.c_int32, P(P(SeqtabMergeOut)), C.c_char_p]
        L.dada2b_merge_seqtabs_free.argtypes = [P(SeqtabMergeOut)]
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


def nwhamming(s1, s2, vec=False, band=-1, match=5, mismatch=-4, gap=-8, homo_gap=None, endsfree=True, device=0):
    """R/misc.R:216-220 (nwalign, then C_eval_pair's mismatch + indel), vectorised over pairs like R's Vectorize:
    strings or equal-length lists of strings; the keyword arguments are nwalign's (R's `...`).  -> int, or int32 array
    for lists."""
    a, b, one = align._pairs(s1, s2, "nwhamming")
    cnt = align.eval_counts(a, b, device=device, match=match, mismatch=mismatch, gap=gap, homo_gap=homo_gap, band=band,
                            endsfree=endsfree, vec=vec)
    out = cnt[:, 1] + cnt[:, 2]
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


# ---- mergeSequenceTables ----------------------------------------------------------------------------------------------
def merge_columns(mats, colnames, row_out, nrow_out, tryRC=False, order_by=1, device=0):
    """dada2b_merge_seqtabs.  mats: int32 [nrow_t, ncol_t] tables; colnames: each table's column names; row_out: the
    output row of every row of every table, concatenated (-1 = skip).  -> (int32 mat [nrow_out, ncol_out], name_src
    int32: the input column, counted over all tables, whose name each output column carries, stats dict)."""
    mats = [np.ascontiguousarray(m, dtype=np.int32) for m in mats]
    flat = [c.encode() for cols in colnames for c in cols]
    lens = np.fromiter((len(c) for c in flat), np.int64, len(flat))
    name_off = np.zeros(len(flat) + 1, np.int64)
    np.cumsum(lens, out=name_off[1:])
    names = b"".join(flat)
    nrow = np.array([m.shape[0] for m in mats], np.int32)
    ncol = np.array([m.shape[1] for m in mats], np.int32)
    row_out = np.ascontiguousarray(row_out, dtype=np.int32)
    entries = np.concatenate([m.ravel() for m in mats]) if mats else np.zeros(0, np.int32)
    if len(row_out) != int(nrow.sum()) or len(flat) != int(ncol.sum()):
        raise api.Dada2bError("dada2b: row_out / colnames do not match the tables.")
    L = _lib()
    a = SeqtabMergeIn(len(mats), nrow.ctypes.data, ncol.ctypes.data, names, name_off.ctypes.data, row_out.ctypes.data,
                      entries.ctypes.data, int(nrow_out), int(bool(tryRC)), int(order_by))
    out = C.POINTER(SeqtabMergeOut)()
    eb = C.create_string_buffer(ERRLEN)
    if L.dada2b_merge_seqtabs(C.byref(a), int(device), C.byref(out), eb):
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        nc = r.ncol_out
        mat = np.ctypeslib.as_array(r.mat, shape=(int(nrow_out) * nc,)).reshape(int(nrow_out), nc).copy()
        src = np.ctypeslib.as_array(r.name_src, shape=(nc,)).copy()
        return mat, src, {k: getattr(r, k) for k in MERGE_STATS}
    finally:
        L.dada2b_merge_seqtabs_free(out)


def _file_name(x):
    return isinstance(x, (str, bytes, os.PathLike))


def _table_problem(tab):
    """is.sequence.table (R/multiSample.R:206-238) on a (mat, colnames, rownames) table: the warning of the first check
    it fails, or None; duplicated names only warn.  R drops zero-length dimnames, so a table without columns has no
    column names (and one without rows no row names)."""
    if not isinstance(tab, (tuple, list)) or len(tab) != 3:
        return "Not a matrix."
    mat, cols, rows = tab
    mat = np.asarray(mat)
    if mat.ndim != 2 or not (np.issubdtype(mat.dtype, np.number) or mat.dtype == np.bool_):
        return "Not a matrix."
    for names, n, what in ((cols, mat.shape[1], "colnames"), (rows, mat.shape[0], "rownames")):
        if names is not None and len(names) != n:
            raise api.Dada2bError("dada2b: a table's %s do not match its shape %s." % (what, mat.shape))
    if (mat < 0).any():
        return "Negative entries."
    if cols is None or mat.shape[1] == 0:
        return "Column (sequence) names are missing."
    if rows is None or mat.shape[0] == 0:
        return "Row (sample) names are missing."
    if any(len(c) == 0 for c in cols):
        return "Some column (sequence) names are blank."
    if any(len(str(r)) == 0 for r in rows):
        return "Some row (sample) names are blank."
    if len(set(cols)) < len(cols):
        warnings.warn("Duplicated column (sequences) names.")
    if len(set(rows)) < len(rows):
        warnings.warn("Duplicated row (sample) names.")
    return None


def _int32_entries(mat):
    mat = np.asarray(mat)
    if mat.dtype == np.bool_:
        return mat.astype(np.int32)
    if not np.issubdtype(mat.dtype, np.integer):
        if not np.isfinite(mat).all() or (mat != np.floor(mat)).any():
            raise api.Dada2bError("dada2b: sequence table entries must be whole numbers.")
    if mat.size and mat.max() > np.iinfo(np.int32).max:
        raise api.Dada2bError("dada2b: a table entry exceeds the int32 range (R would return NA).")
    return mat.astype(np.int32)


def _merge_inputs(table1, table2, more, tables, repeats):
    """R/multiSample.R:290-320: the tables, their validation and the sample names.  -> (tables, sample names,
    row_out): row_out[t][i] is the output row of row i of table t, or -1 when a later row of table t has the same name
    (R's sub-assignment: the last one wins)."""
    if tables is None and (table1 is None or table2 is None):
        raise api.Dada2bError("Either 'tables' or 'table1' and 'table2' must be provided.")
    names = None
    if tables is not None:
        if _file_name(tables) or (isinstance(tables, (list, tuple, dict)) and any(_file_name(t) for t in
                                                                                  (tables.values() if isinstance(tables, dict) else tables))):
            raise api.Dada2bError("dada2b: tables given as RDS file names are not supported (there is no RDS reader); pass the tables.")
        if isinstance(tables, dict):
            names, tables = [str(k) for k in tables], list(tables.values())
        elif isinstance(tables, (list, tuple)):
            tables = list(tables)
        else:
            raise api.Dada2bError("'tables' must be a list or vector.")
    else:
        tables = [table1, table2] + list(more)
    if len(tables) < 2:
        raise api.Dada2bError("At least two sequence tables are expected")
    problems = [_table_problem(t) for t in tables]
    for p in problems:
        if p is not None:
            warnings.warn(p)
    if any(p is not None for p in problems):
        bad = ", ".join(names[i] for i, p in enumerate(problems) if p is not None) if names else ""
        raise api.Dada2bError("Some sequence tables found invalid" + (": " + bad if bad else ""))
    index, dups = {}, {}
    for t in tables:
        for r in t[2]:
            if r in index:
                dups[r] = None
            else:
                index[r] = len(index)
    if dups:
        if repeats == "error":
            raise api.Dada2bError("Duplicated sample names detected in the sequence table row names: " + ", ".join(map(str, dups)))
        print("Duplicated sample names detected in the sequence table row names.", file=sys.stderr)
    row_out = []
    for t in tables:
        rows = list(t[2])
        last = {r: i for i, r in enumerate(rows)}
        row_out.append(np.array([index[r] if last[r] == i else -1 for i, r in enumerate(rows)], np.int32))
    return tables, list(index), row_out


def mergeSequenceTables(table1=None, table2=None, *more, tables=None, repeats="error", orderBy="abundance", tryRC=False, device=0):
    """R/multiSample.R:290-364.  Tables are (mat, colnames, rownames), as makeSequenceTable returns them, given as
    table1, table2, ... or as `tables` (a list, or a dict whose keys name the tables in the invalid-table message).
    repeats="error" refuses a sample name that occurs twice (across tables or within one); any other value merges
    them, in first-occurrence order.  tryRC re-orients a sequence whose reverse complement occurs earlier.  orderBy:
    "abundance", "nsamples", or None / any other string for first-seen order.  Entries must be whole numbers >= 0 and
    column names upper-case IUPAC (ACGTMRWSYKVHDBN); RDS file names are refused.  -> (int32 mat [nsample, nseq],
    colnames, rownames)."""
    tables, rownames, row_out = _merge_inputs(table1, table2, more, tables, repeats)
    mats = [_int32_entries(t[0]) for t in tables]
    cols = [list(t[1]) for t in tables]
    order = ORDER_BY.get(orderBy, 0) if isinstance(orderBy, str) else 0
    mat, src, st = merge_columns(mats, cols, np.concatenate(row_out), len(rownames), tryRC, order, device)
    if st["n_rc"] > 0:
        print("Reverse complemented sequences detected and re-oriented.", file=sys.stderr)
    flat = [c for cs in cols for c in cs]
    return mat, [flat[k] for k in src], rownames

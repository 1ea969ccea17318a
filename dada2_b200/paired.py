"""mergePairs (R/paired.R:92-202): merge denoised forward and reverse reads, sample by sample.

The work runs in libdada2b.so behind include/dada2b_merge.h (`dada2b_merge_samples`): per-read cluster lookup, the
tabulation of the unique (forward, reverse) pairings and their order on the device, one alignment per distinct (forward
sequence, reverse sequence, prefer) across all samples, the accept rule and the blanking of rejected sequences.  This module
restates the R around it (argument forms and messages, scores, nwalign's `...`, propagateCol, returnRejects, the verbose
and duplicate messages, the return shape) and only marshals.  No CPU fallback.

A merger is a dict of columns, in R's order: sequence (list of str), abundance, forward, reverse, nmatch, nmismatch, nindel,
prefer (int32; NA_INT under justConcatenate), accept (bool), then F.<col> / R.<col> for propagateCol.
"""
import ctypes as C
import os
import sys

import numpy as np

from . import api
from .merge import MergeOpts

ERRLEN = 256
NA_INT = np.iinfo(np.int32).min
COLS = ("sequence", "abundance", "forward", "reverse", "nmatch", "nmismatch", "nindel", "prefer", "accept")
STATS = ("n_reads", "n_pairings", "n_aligned", "n_batches", "n_cells", "gpu_launches", "h2d_bytes", "d2h_bytes", "ms_k_tab",
         "ms_k_merge", "ms_total")


class PairsIn(C.Structure):
    _fields_ = [("nsamples", C.c_int32), ("nreadsF", C.c_void_p), ("nreadsR", C.c_void_p), ("mapF", C.c_void_p), ("mapR", C.c_void_p),
                ("nuniqF", C.c_void_p), ("nuniqR", C.c_void_p), ("dmapF", C.c_void_p), ("dmapR", C.c_void_p),
                ("nclustF", C.c_void_p), ("nclustR", C.c_void_p), ("n0F", C.c_void_p), ("n0R", C.c_void_p),
                ("seqF", C.c_char_p), ("seqR", C.c_char_p), ("seqF_off", C.c_void_p), ("seqR_off", C.c_void_p)]


class PairsOpts(C.Structure):
    _fields_ = [("align", MergeOpts), ("min_overlap", C.c_int32), ("max_mismatch", C.c_int32), ("just_concatenate", C.c_int32)]


class PairsOut(C.Structure):
    _fields_ = [("nsamples", C.c_int32), ("pair_off", C.POINTER(C.c_int64)), ("forward", C.POINTER(C.c_int32)),
                ("reverse", C.POINTER(C.c_int32)), ("abundance", C.POINTER(C.c_int32)), ("nmatch", C.POINTER(C.c_int32)),
                ("nmismatch", C.POINTER(C.c_int32)), ("nindel", C.POINTER(C.c_int32)), ("prefer", C.POINTER(C.c_int32)),
                ("accept", C.POINTER(C.c_uint8)), ("cons_concat", C.POINTER(C.c_char)), ("cons_off", C.POINTER(C.c_int64))] + \
               [(k, C.c_int64) for k in STATS[:8]] + [(k, C.c_double) for k in STATS[8:]]


_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_merge_samples.argtypes = [P(PairsIn), P(PairsOpts), C.c_int32, P(P(PairsOut)), C.c_char_p]
        L.dada2b_merge_samples_free.argtypes = [P(PairsOut)]
        _BOUND = True
    return L


def _cat_i32(arrs):
    return np.ascontiguousarray(np.concatenate([np.asarray(a).ravel() for a in arrs]) if arrs else np.zeros(0), dtype=np.int32)


def _cat_seqs(lists):
    seqs = [x for sq in lists for x in sq]
    lens = np.fromiter((len(x) for x in seqs), dtype=np.int64, count=len(seqs))
    off = np.zeros(len(seqs) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    return "".join(seqs).encode(), off


def merge_samples(mapF, mapR, dmapF, dmapR, seqF, seqR, n0F, n0R, minOverlap=12, maxMismatch=0, justConcatenate=False, match=1,
                  mismatch=-64, gap=-64, homo_gap=None, trimOverhang=False, device=0, return_stats=False):
    """dada2b_merge_samples over S samples: per-sample lists of derep maps (mapF / mapR), dada maps (dmapF / dmapR), cluster
    sequences (seqF; seqR as dada() reports them, not reverse-complemented) and clustering n0.  -> list of S dicts with
    forward, reverse, abundance, nmatch, nmismatch, nindel, prefer (0 under justConcatenate), accept and sequence ("" where
    rejected), pairings in R's order; with return_stats also the work counters and timings."""
    S = len(mapF)
    if not all(len(x) == S for x in (mapR, dmapF, dmapR, seqF, seqR, n0F, n0R)):
        raise api.Dada2bError("dada2b: every per-sample input needs one entry per sample.")
    L = _lib()
    mF, mR = [np.asarray(m).ravel() for m in mapF], [np.asarray(m).ravel() for m in mapR]
    dF, dR = [np.asarray(m).ravel() for m in dmapF], [np.asarray(m).ravel() for m in dmapR]
    nrF = np.array([len(m) for m in mF], np.int64)
    nrR = np.array([len(m) for m in mR], np.int64)
    nuF = np.array([len(m) for m in dF], np.int32)
    nuR = np.array([len(m) for m in dR], np.int32)
    ncF = np.array([len(x) for x in seqF], np.int32)
    ncR = np.array([len(x) for x in seqR], np.int32)
    if any(len(a) != n for a, n in zip(n0F, ncF)) or any(len(a) != n for a, n in zip(n0R, ncR)):
        raise api.Dada2bError("dada2b: clustering$n0 needs one entry per cluster sequence.")
    cmF, cmR, cdF, cdR, c0F, c0R = _cat_i32(mF), _cat_i32(mR), _cat_i32(dF), _cat_i32(dR), _cat_i32(n0F), _cat_i32(n0R)
    bF, oF = _cat_seqs(seqF)
    bR, oR = _cat_seqs(seqR)
    inp = PairsIn(S, nrF.ctypes.data, nrR.ctypes.data, cmF.ctypes.data, cmR.ctypes.data, nuF.ctypes.data, nuR.ctypes.data,
                  cdF.ctypes.data, cdR.ctypes.data, ncF.ctypes.data, ncR.ctypes.data, c0F.ctypes.data, c0R.ctypes.data,
                  bF, bR, oF.ctypes.data, oR.ctypes.data)
    hg = gap if homo_gap is None else homo_gap
    o = PairsOpts(MergeOpts(int(match), int(mismatch), int(gap), int(hg), -1, int(bool(trimOverhang))), int(minOverlap), int(maxMismatch),
                  int(bool(justConcatenate)))
    out = C.POINTER(PairsOut)()
    eb = C.create_string_buffer(ERRLEN)
    rc = L.dada2b_merge_samples(C.byref(inp), C.byref(o), int(device), C.byref(out), eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        po = np.ctypeslib.as_array(r.pair_off, shape=(S + 1,)).copy()
        n = int(po[-1])
        n1 = max(n, 1)

        def arr(p, dt=np.int32):
            return np.ctypeslib.as_array(p, shape=(n1,))[:n].astype(dt)
        cols = {k: arr(getattr(r, k)) for k in ("forward", "reverse", "abundance", "nmatch", "nmismatch", "nindel", "prefer")}
        cols["accept"] = arr(r.accept, bool)
        co = np.ctypeslib.as_array(r.cons_off, shape=(n + 1,)).copy()
        raw = C.string_at(r.cons_concat, int(co[-1])).decode() if n else ""
        seqs = [raw[co[x]:co[x + 1]] for x in range(n)]
        res = []
        for k in range(S):
            a, b = int(po[k]), int(po[k + 1])
            d = {c: v[a:b].copy() for c, v in cols.items()}
            d["sequence"] = seqs[a:b]
            res.append(d)
        if return_stats:
            return res, {k: getattr(r, k) for k in STATS}
        return res
    finally:
        L.dada2b_merge_samples_free(out)


def _is_dada(x):
    return isinstance(x, dict) and "clustering" in x and "map" in x


def _is_derep(x):
    return isinstance(x, dict) and "uniques" in x and "map" in x


def _listify(x, one):
    """-> (list, names or None, single?)"""
    if one(x):
        return [x], None, True
    if isinstance(x, dict):
        return list(x.values()), list(x.keys()), False
    if isinstance(x, (str, os.PathLike)):
        return [x], None, True
    if isinstance(x, (list, tuple)):
        return list(x), None, False
    return None, None, False


def _nwalign_opts(maxMismatch, nw):
    """paired.R:153-159: MATCH 1, MISMATCH = GAP = -64 (maxMismatch 0) or -8, then nwalign(x, y, band=-1, ...)."""
    mm = -64 if maxMismatch == 0 else -8
    o = dict(match=1, mismatch=mm, gap=mm, homo_gap=None)
    for k, v in nw.items():
        if k == "band":
            raise TypeError('formal argument "band" matched by multiple actual arguments')
        if k == "vec":
            if v:
                raise ValueError("nwalign(vec = TRUE) is not supported by mergePairs here: only the endsfree aligner runs on the GPU.")
        elif k == "endsfree":
            if not v:
                raise ValueError("nwalign(endsfree = FALSE) is not supported by mergePairs here: only the endsfree aligner runs on the GPU.")
        elif k in o:
            o[k] = v
        else:
            raise TypeError("unused argument (%s)" % k)
    return o


def _empty():
    d = {c: np.zeros(0, np.int32) for c in COLS}
    d["sequence"] = []
    d["accept"] = np.zeros(0, bool)
    return d


def mergePairs(dadaF, derepF, dadaR, derepR, minOverlap=12, maxMismatch=0, returnRejects=False, propagateCol=(), justConcatenate=False,
               trimOverhang=False, verbose=False, device=0, return_stats=False, **nwalign_opts):
    """mergePairs (R/paired.R:92-202).  dadaF / dadaR: a dada() result, a list of them or a dict name -> result; derepF /
    derepR: derep dicts or fastq paths in the same form (paths are dereplicated on the device).  `nwalign_opts` are nwalign's
    arguments (match, mismatch, gap, homo_gap), as R's `...`.  -> one merger for one sample, else a list (or a dict keyed
    like dadaF) of mergers; with return_stats, (that, stats of the native call)."""
    from .derep import derepFastq
    dF, names, oneF = _listify(dadaF, _is_dada)
    dR, _, _ = _listify(dadaR, _is_dada)
    rF, _, _ = _listify(derepF, _is_derep)
    rR, _, _ = _listify(derepR, _is_derep)
    if dF is None or dR is None or not all(_is_dada(x) for x in dF + dR):
        raise ValueError("dadaF and dadaR must be provided as dada-class objects or lists of dada-class objects.")

    def derep_ok(v):
        return v is not None and (all(_is_derep(x) for x in v) or all(isinstance(x, (str, os.PathLike)) for x in v))
    if not (derep_ok(rF) and derep_ok(rR)):
        raise ValueError("derepF and derepR must be provided as derep-class objects or as character vectors of filenames.")
    if len({len(dF), len(rF), len(dR), len(rR)}) > 1:
        raise ValueError("The dadaF/derepF/dadaR/derepR arguments must be the same length.")
    o = _nwalign_opts(maxMismatch, nwalign_opts)
    rF = [x if isinstance(x, dict) else derepFastq(x, device=device) for x in rF]
    rR = [x if isinstance(x, dict) else derepFastq(x, device=device) for x in rR]
    for x in rF + rR:
        m = np.asarray(x["map"])
        if not np.issubdtype(m.dtype, np.integer):
            raise ValueError("Incorrect format of $map in derep-class arguments.")
    clF = [d["clustering"] for d in dF]
    clR = [d["clustering"] for d in dR]
    got = merge_samples([x["map"] for x in rF], [x["map"] for x in rR], [d["map"] for d in dF], [d["map"] for d in dR],
                        [list(c["sequence"]) for c in clF], [list(c["sequence"]) for c in clR], [c["n0"] for c in clF],
                        [c["n0"] for c in clR], minOverlap=minOverlap, maxMismatch=maxMismatch, justConcatenate=justConcatenate,
                        trimOverhang=trimOverhang, device=device, return_stats=return_stats, **o)
    if return_stats:
        got, stats = got
    rval = []
    for i, g in enumerate(got):
        nreads = len(rF[i]["map"])
        if len(g["forward"]) == 0:                                 # paired.R:128-136
            if verbose:
                print("No paired-reads (in ZERO unique pairings) successfully merged out of %d pairings) input." % nreads, file=sys.stderr)
            rval.append(_empty())
            continue
        m = {"sequence": g["sequence"]}
        for c in COLS[1:]:
            m[c] = g[c]
        if justConcatenate:
            m["prefer"] = np.full(len(g["prefer"]), NA_INT, np.int32)
        for col in [c for c in propagateCol if c in clF[i]]:        # paired.R:179-183
            for tag, cl, idx in (("F.", clF[i], g["forward"]), ("R.", clR[i], g["reverse"])):
                v = cl[col]
                m[tag + col] = [v[k - 1] for k in idx] if isinstance(v, list) else np.asarray(v)[idx - 1]
        acc = m["accept"]
        if verbose:
            ab = m["abundance"].astype(np.int64)
            print("%d paired-reads (in %d unique pairings) successfully merged out of %d (in %d pairings) input." % (
                ab[acc].sum(), acc.sum(), ab.sum(), len(ab)), file=sys.stderr)
        if not returnRejects:
            m = {k: ([x for x, a in zip(v, acc) if a] if isinstance(v, list) else v[acc]) for k, v in m.items()}
        if len(set(m["sequence"])) < len(m["sequence"]):
            print("Duplicate sequences in merged output.", file=sys.stderr)
        rval.append(m)
    if names is not None and not (oneF and len(rval) == 1):
        rval = dict(zip(names, rval))
    if len(rval) == 1:
        rval = next(iter(rval.values())) if isinstance(rval, dict) else rval[0]
    return (rval, stats) if return_stats else rval

"""Primer removal for the GPU path: removePrimers (R/filter.R:81-233).

The matching block (four vmatchPattern scans per read, the choice of hits, orientation, the keep and trim rules) runs in
libdada2b.so behind include/dada2b_primer.h, one call per file.  This module checks arguments, parses and writes fastq
on the host (filter.py's reader and writer) and marshals; no CPU fallback.  `remove_primers_reads` is the in-memory
form: its survivors go straight into derep.derep_reads.
"""
import ctypes as C
import os

import numpy as np

from . import api
from .derep import DerepIn
from .filter import ERRLEN, Reads, _as_reads, _remove, _write, fastq_bytes, read_fastq_records

REASONS = ("kept", "no forward hit", "no reverse hit", "empty window", "file skipped")
FLIPPED, MULTI_FWD, MULTI_REV = 1, 2, 4
MAXLEN = 64


class PrimerOpts(C.Structure):
    _fields_ = [("primer_fwd", C.c_char_p), ("primer_rev", C.c_char_p), ("max_mismatch", C.c_int32), ("allow_indels", C.c_int32),
                ("trim_fwd", C.c_int32), ("trim_rev", C.c_int32), ("orient", C.c_int32), ("reserved", C.c_int32)]


class PrimerOut(C.Structure):
    _fields_ = [("nreads", C.c_int32), ("nout", C.c_int32), ("skipped", C.c_int32), ("multi", C.c_int32),
                ("reason", C.POINTER(C.c_uint8)), ("flags", C.POINTER(C.c_uint8)), ("src", C.POINTER(C.c_int32)),
                ("seq_concat", C.c_void_p), ("seq_off", C.c_void_p), ("qual_concat", C.c_void_p), ("gpu_launches", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64), ("ms_h2d", C.c_double),
                ("ms_kernels", C.c_double), ("ms_d2h", C.c_double), ("ms_device", C.c_double), ("ms_total", C.c_double)]


class Hit(C.Structure):
    _fields_ = [("count", C.c_int32), ("first_start", C.c_int32), ("first_end", C.c_int32), ("last_start", C.c_int32),
                ("last_end", C.c_int32)]


HIT_DTYPE = np.dtype([(k, np.int32) for k in ("count", "first_start", "first_end", "last_start", "last_end")])
STATS = ("gpu_launches", "h2d_bytes", "d2h_bytes", "kernel_bytes", "ms_h2d", "ms_kernels", "ms_d2h", "ms_device", "ms_total")

_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_primer_default_opts.argtypes = [P(PrimerOpts)]
        L.dada2b_remove_primers.argtypes = [P(DerepIn), P(PrimerOpts), C.c_int32, P(P(PrimerOut)), C.c_char_p]
        L.dada2b_primer_free.argtypes = [P(PrimerOut)]
        L.dada2b_test_primer_hits.argtypes = [P(DerepIn), P(PrimerOpts), C.c_int32, C.c_void_p, C.c_char_p]
        _BOUND = True
    return L


def _opts(primer_fwd, primer_rev, max_mismatch, allow_indels, trim_fwd, trim_rev, orient):
    for p in (primer_fwd,) + ((primer_rev,) if primer_rev is not None else ()):
        if not isinstance(p, str):
            raise api.Dada2bError("Primer sequences must be provided as base R strings.")
    if isinstance(max_mismatch, bool) or max_mismatch != int(max_mismatch):
        raise api.Dada2bError("dada2b: max.mismatch must be a whole number (got %r)." % (max_mismatch,))
    o = PrimerOpts()
    _lib().dada2b_primer_default_opts(C.byref(o))
    o.primer_fwd = primer_fwd.encode()
    o.primer_rev = primer_rev.encode() if primer_rev is not None else None
    o.max_mismatch = int(max_mismatch)
    o.allow_indels = int(bool(allow_indels))
    o.trim_fwd, o.trim_rev, o.orient = int(bool(trim_fwd)), int(bool(trim_rev)), int(bool(orient))
    return o


def _run(reads, opts, device):
    L = _lib()
    out = C.POINTER(PrimerOut)()
    eb = C.create_string_buffer(ERRLEN)
    ri = reads.c_in()
    if L.dada2b_remove_primers(C.byref(ri), C.byref(opts), int(device), C.byref(out), eb):
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        n, k = r.nreads, r.nout
        off = np.ctypeslib.as_array(C.cast(r.seq_off, C.POINTER(C.c_int64)), shape=(k + 1,)).copy()
        nb = int(off[-1])
        return {"reason": np.ctypeslib.as_array(r.reason, shape=(max(n, 1),))[:n].copy(),
                "flags": np.ctypeslib.as_array(r.flags, shape=(max(n, 1),))[:n].copy(),
                "src": np.ctypeslib.as_array(r.src, shape=(max(k, 1),))[:k].copy(),
                "skipped": bool(r.skipped), "multi": bool(r.multi),
                "reads": Reads(C.string_at(r.seq_concat, nb), off, np.frombuffer(C.string_at(r.qual_concat, nb), dtype=np.uint8).copy()),
                "stats": {s: getattr(r, s) for s in STATS}}
    finally:
        L.dada2b_primer_free(out)


def remove_primers_reads(seqs, quals, primer_fwd, primer_rev=None, max_mismatch=2, allow_indels=False, trim_fwd=True, trim_rev=True,
                         orient=True, device=0):
    """The matching block of removePrimers on one file's reads in memory.
    seqs: list[str] (upper-case IUPAC) or a filter.Reads; quals: numeric qualities (list of arrays or one uint8 array).
    -> dict(seqs, quals: the kept reads, oriented and trimmed, in derep_reads' input form; reads: the same as a Reads;
    reason: uint8[nreads] (index in REASONS); flags: uint8[nreads] (FLIPPED, MULTI_FWD, MULTI_REV); src: int32[nout] input
    index of each kept read; skipped: R skips the whole file; multi: R's "Multiple matches" condition; stats)."""
    rd = _as_reads(seqs, quals)
    r = _run(rd, _opts(primer_fwd, primer_rev, max_mismatch, allow_indels, trim_fwd, trim_rev, orient), device)
    r["seqs"], r["quals"] = r["reads"].strings(), r["reads"].qual
    return r


def test_primer_hits(seqs, quals, primer_fwd, primer_rev=None, max_mismatch=2, orient=True, device=0):
    """Hit hook: HIT_DTYPE[nreads, 4] for the scans (forward, reverse) x (read, reverse complement), 1-based coordinates of
    the scanned sequence, from dada2b_remove_primers' own launch sequence."""
    rd = _as_reads(seqs, quals)
    o = _opts(primer_fwd, primer_rev, max_mismatch, False, True, True, orient)
    out = np.zeros((max(len(rd), 1), 4), HIT_DTYPE)
    eb = C.create_string_buffer(ERRLEN)
    ri = rd.c_in()
    if _lib().dada2b_test_primer_hits(C.byref(ri), C.byref(o), int(device), out.ctypes.data, eb):
        raise api.Dada2bError(eb.value.decode())
    return out[:len(rd)]


test_primer_hits.__test__ = False


def _filt_print(nin, nout):
    # filt.print (R/filter.R:235-239); R's round() goes half to even, as Python's does
    pct = "NaN" if nin == 0 else ("%s" % round(nout * 100 / nin, 1)).rstrip("0").rstrip(".")
    print("Read in %d, output %d (%s%%) filtered sequences." % (nin, nout, pct))


def removePrimers(fn, fout, primer_fwd, primer_rev=None, max_mismatch=2, allow_indels=False, trim_fwd=True, trim_rev=True, orient=True,
                  compress=True, verbose=False, device=0):
    """R/filter.R:81-233 -> int64 [files x 2] matrix of (reads.in, reads.out), one row per input file in order.
    A skipped file (no read has a forward hit as read, or none a reverse hit) gets no output file, as in R."""
    fn = [fn] if isinstance(fn, (str, os.PathLike)) else list(fn)
    fout = [fout] if isinstance(fout, (str, os.PathLike)) else list(fout)
    if len(fn) != len(fout):
        raise api.Dada2bError("Every input file must have a corresponding output file.")
    if allow_indels:
        raise api.Dada2bError("dada2b: allow.indels=TRUE is not supported (Biostrings' choice among equal-edit placements is not "
                              "restated).")
    for d in dict.fromkeys(os.path.dirname(os.path.abspath(p)) for p in fout):
        if not os.path.isdir(d):
            print("Creating output directory: " + d)
            os.makedirs(d, exist_ok=True)
    if not all(os.path.exists(f) for f in fn):
        raise api.Dada2bError("Some input files do not exist.")
    ins = [os.path.realpath(p) for p in fn]
    outs = [os.path.abspath(p) for p in fout]
    if len(set(outs)) != len(outs):
        raise api.Dada2bError("All output files must be distinct.")
    if set(outs) & set(ins):
        raise api.Dada2bError("Output files must be distinct from the input files.")
    o = _opts(primer_fwd, primer_rev, max_mismatch, allow_indels, trim_fwd, trim_rev, orient)
    rows = []
    first_multi = True
    for path, op in zip(fn, fout):
        ids, reads = read_fastq_records(path)
        r = _run(reads, o, device)
        if r["skipped"]:
            _filt_print(len(reads), 0)
            rows.append((len(reads), 0))
            continue
        if r["multi"] and verbose and first_multi:
            print("Multiple matches to the primer(s) in some sequences. Using the longest possible match.")
            first_multi = False
        nflip = int(np.count_nonzero(r["flags"] & FLIPPED))
        if orient and nflip and verbose:
            print(nflip, "sequences out of", len(reads), "are being reverse-complemented.")
        if os.path.exists(op):
            _remove(op)
            if verbose:
                print("Overwriting file:" + op)
        _write(op, fastq_bytes([ids[i] for i in r["src"]], r["reads"]), compress)
        rows.append((len(reads), len(r["src"])))
        if verbose:
            _filt_print(len(reads), len(r["src"]))
    rval = np.array(rows, dtype=np.int64).reshape(len(fn), 2)
    if np.all(rval[:, 1] == 0):
        import warnings
        warnings.warn("No reads passed the primer detection.")
    elif np.any(rval[:, 1] == 0):
        print("Some input samples had no reads pass the primer detection.")
    return rval

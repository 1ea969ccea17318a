"""Read filtering for the GPU path: filterAndTrim, fastqFilter and fastqPairedFilter (R/filter.R:402-497, :613-730,
:878-1141), isPhiX, seqComplexity and C_matchRef.

Stages 1-12 of the reference's per-chunk loop (orient.fwd, maxLen, trimLeft, trimRight, truncQ, truncLen, minLen, maxN,
minQ, maxEE, rm.phix, rm.lowcomplex) run in libdada2b.so behind include/dada2b_filter.h, for all chunks of a file in one
call.  This module parses and writes fastq on the host and marshals; no CPU fallback.  `filter_reads` is the in-memory
form: its survivors go straight into derep.derep_reads.

The phiX genome is reference data the caller supplies (`phix=`, a FASTA path or the sequence); it is not bundled.
"""
import ctypes as C
import gzip
import math
import os

import numpy as np

from . import api
from .derep import DerepIn

ERRLEN = 256
REASONS = ("kept", "orient.fwd", "maxLen", "trimLeft", "trimRight", "truncQ", "truncLen", "minLen", "maxN", "minQ", "maxEE",
           "rm.phix", "rm.lowcomplex")
MATE1, MATE2, FLIPPED = 1, 2, 4
IUPAC = "ACGTRYSWKMBDHVN"


class MateOpts(C.Structure):
    _fields_ = [("trunc_q", C.c_int32), ("trunc_len", C.c_int32), ("trim_left", C.c_int32), ("trim_right", C.c_int32),
                ("max_len", C.c_int32), ("min_len", C.c_int32), ("max_n", C.c_int32), ("min_q", C.c_int32), ("max_ee", C.c_double),
                ("rm_phix", C.c_int32), ("reserved", C.c_int32), ("rm_lowcomplex", C.c_double)]


class FilterOpts(C.Structure):
    _fields_ = [("mate", MateOpts * 2), ("orient_fwd", C.c_char_p), ("phix", C.c_char_p), ("chunk_n", C.c_int64)]


class FilterOut(C.Structure):
    _fields_ = [("nreads", C.c_int32), ("nout", C.c_int32), ("paired", C.c_int32), ("reason", C.POINTER(C.c_uint8)),
                ("flags", C.POINTER(C.c_uint8)), ("src", C.POINTER(C.c_int32)), ("seq_concat", C.c_void_p * 2),
                ("seq_off", C.c_void_p * 2), ("qual_concat", C.c_void_p * 2), ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64),
                ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64), ("ms_h2d", C.c_double), ("ms_kernels", C.c_double),
                ("ms_d2h", C.c_double), ("ms_device", C.c_double), ("ms_total", C.c_double)]


class Stage(C.Structure):
    _fields_ = [("trim_fail", C.c_int32), ("flipped", C.c_int32), ("start", C.c_int32), ("end", C.c_int32), ("n_other", C.c_int32),
                ("min_q", C.c_int32), ("hits_fwd", C.c_int32), ("hits_rc", C.c_int32), ("ee", C.c_double), ("complexity", C.c_double)]


STAGE_DTYPE = np.dtype([(k, np.int32) for k in ("trim_fail", "flipped", "start", "end", "n_other", "min_q", "hits_fwd", "hits_rc")]
                       + [("ee", np.float64), ("complexity", np.float64)])
STATS = ("gpu_launches", "h2d_bytes", "d2h_bytes", "kernel_bytes", "ms_h2d", "ms_kernels", "ms_d2h", "ms_device", "ms_total")

_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_filter_default_opts.argtypes = [P(FilterOpts)]
        L.dada2b_filter.argtypes = [P(DerepIn), P(DerepIn), P(FilterOpts), C.c_int32, P(P(FilterOut)), C.c_char_p]
        L.dada2b_filter_free.argtypes = [P(FilterOut)]
        L.dada2b_match_ref.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_char_p]
        L.dada2b_seq_complexity.argtypes = [C.c_int32, C.c_char_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_char_p]
        L.dada2b_test_filter_stages.argtypes = [P(DerepIn), P(FilterOpts), C.c_int32, C.c_void_p, C.c_char_p]
        _BOUND = True
    return L


# ---- marshalling ------------------------------------------------------------------------------------------------------
class Reads:
    """One read set in dada2b_derep_in's layout: seq (bytes), off (int64[n+1]), qual (uint8[off[-1]])."""

    def __init__(self, seq, off, qual):
        self.seq, self.off, self.qual = seq, np.ascontiguousarray(off, dtype=np.int64), np.ascontiguousarray(qual, dtype=np.uint8)
        if len(self.qual) != self.off[-1] or len(self.seq) != self.off[-1]:
            raise api.Dada2bError("dada2b: qualities and sequences have different lengths.")

    @classmethod
    def from_lists(cls, seqs, quals):
        lens = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=len(seqs))
        off = np.zeros(len(seqs) + 1, np.int64)
        np.cumsum(lens, out=off[1:])
        if isinstance(quals, np.ndarray) and quals.ndim == 1:
            q = quals
        else:
            q = np.concatenate([np.asarray(x, dtype=np.uint8).ravel() for x in quals]) if len(seqs) else np.zeros(0, np.uint8)
        return cls("".join(seqs).encode(), off, q)

    def __len__(self):
        return len(self.off) - 1

    def strings(self):
        s = self.seq.decode()
        o = self.off
        return [s[o[i]:o[i + 1]] for i in range(len(self))]

    def c_in(self, chunk_n=0):
        return DerepIn(len(self), self.seq, self.off.ctypes.data, self.qual.ctypes.data, int(chunk_n))


def _pack_any(seqs):
    if isinstance(seqs, str):
        seqs = [seqs]
    seqs = list(seqs)
    lens = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=len(seqs))
    off = np.zeros(len(seqs) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    buf = "".join(seqs).encode("latin-1")
    if len(buf) != off[-1]:
        raise api.Dada2bError("dada2b: sequences must be single-byte text.")
    return seqs, buf, off


def _pair(v, name, paired):
    if isinstance(v, (list, tuple, np.ndarray)):
        v = list(v)
        if len(v) == 1:
            v = v * 2
        if not paired and len(v) != 2:
            raise api.Dada2bError("Filtering and trimming arguments should be of length 1 when processing single-end (rather than "
                                  "paired-end) data.")
        if len(v) != 2:
            raise api.Dada2bError("Input variable %s must be length 1 or 2 (Forward, Reverse)." % name)
        if not paired and v[0] != v[1]:
            raise api.Dada2bError("Filtering and trimming arguments should be of length 1 when processing single-end (rather than "
                                  "paired-end) data.")
        return v
    return [v, v]


def _int(v, name, inf=None):
    if inf is not None and v == math.inf:
        return inf
    if isinstance(v, bool) or v != int(v):
        raise api.Dada2bError("dada2b: %s must be a whole number here (got %r)." % (name, v))
    return int(v)


def _phix_seq(phix):
    if phix is None:
        return None
    if isinstance(phix, bytes):
        phix = phix.decode()
    if os.path.exists(str(phix)):
        op = gzip.open if str(phix).endswith(".gz") else open
        with op(phix, "rt") as f:
            lines = [ln.strip() for ln in f]
        body = [ln for ln in lines[1:] if ln and not ln.startswith(">")] if lines and lines[0].startswith(">") else lines
        return "".join(body)
    return str(phix)


def _opts(paired, truncQ, truncLen, trimLeft, trimRight, maxLen, minLen, maxN, minQ, maxEE, rm_phix, rm_lowcomplex, orient_fwd, phix, n):
    o = FilterOpts()
    _lib().dada2b_filter_default_opts(C.byref(o))
    vals = {k: _pair(v, k, paired) for k, v in dict(truncQ=truncQ, truncLen=truncLen, trimLeft=trimLeft, trimRight=trimRight, maxLen=maxLen,
                                                   minLen=minLen, maxN=maxN, minQ=minQ, maxEE=maxEE, rm_phix=rm_phix,
                                                   rm_lowcomplex=rm_lowcomplex).items()}
    for m in range(2):
        mo = o.mate[m]
        mo.trunc_q = _int(vals["truncQ"][m], "truncQ")
        mo.trunc_len = _int(vals["truncLen"][m], "truncLen")
        mo.trim_left = _int(vals["trimLeft"][m], "trimLeft")
        mo.trim_right = _int(vals["trimRight"][m], "trimRight")
        if vals["maxLen"][m] < 0:                           # -1 is the ABI's Inf: a negative maxLen must not turn into "no maximum"
            raise api.Dada2bError("dada2b: maxLen must be >= 0 or Inf (got %r)." % (vals["maxLen"][m],))
        mo.max_len = _int(vals["maxLen"][m], "maxLen", inf=-1)
        mo.min_len = _int(vals["minLen"][m], "minLen")
        mo.max_n = _int(vals["maxN"][m], "maxN")
        mo.min_q = _int(vals["minQ"][m], "minQ")
        mo.max_ee = float(vals["maxEE"][m])
        mo.rm_phix = int(bool(vals["rm_phix"][m]))
        mo.rm_lowcomplex = float(vals["rm_lowcomplex"][m])
    o.orient_fwd = orient_fwd.encode() if orient_fwd is not None else None
    ph = _phix_seq(phix)
    o.phix = ph.encode() if ph is not None else None
    o.chunk_n = int(n)
    tested = [vals["rm_phix"][m] for m in range(2 if paired else 1)]
    if any(tested) and ph is None:
        raise api.Dada2bError("dada2b: rm_phix needs the phiX genome: pass phix= (a FASTA path or the sequence); it is not bundled.")
    return o


def _run(fwd, rev, opts, device):
    L = _lib()
    out = C.POINTER(FilterOut)()
    eb = C.create_string_buffer(ERRLEN)
    fi = fwd.c_in()
    ri = rev.c_in() if rev is not None else None
    rc = L.dada2b_filter(C.byref(fi), C.byref(ri) if ri is not None else None, C.byref(opts), int(device), C.byref(out), eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        n, k = r.nreads, r.nout
        res = {"reason": np.ctypeslib.as_array(r.reason, shape=(max(n, 1),))[:n].copy(),
               "flags": np.ctypeslib.as_array(r.flags, shape=(max(n, 1),))[:n].copy(),
               "src": np.ctypeslib.as_array(r.src, shape=(max(k, 1),))[:k].copy(),
               "stats": {s: getattr(r, s) for s in STATS}}
        mates = []
        for m in range(2 if r.paired else 1):
            off = np.ctypeslib.as_array(C.cast(r.seq_off[m], C.POINTER(C.c_int64)), shape=(k + 1,)).copy()
            nb = int(off[-1])
            seq = C.string_at(r.seq_concat[m], nb)
            qual = np.frombuffer(C.string_at(r.qual_concat[m], nb), dtype=np.uint8).copy()
            mates.append(Reads(seq, off, qual))
        res["mates"] = mates
        return res
    finally:
        L.dada2b_filter_free(out)


def _as_reads(seqs, quals):
    if isinstance(seqs, Reads):
        return seqs
    return Reads.from_lists(list(seqs), quals)


def filter_reads(seqs, quals, rev=None, truncQ=2, truncLen=0, trimLeft=0, trimRight=0, maxLen=math.inf, minLen=20, maxN=0, minQ=0,
                 maxEE=math.inf, rm_phix=True, rm_lowcomplex=0, orient_fwd=None, phix=None, n=1e5, device=0):
    """Stages 1-12 of fastqFilter / fastqPairedFilter on reads in memory, all chunks of n reads in one call.
    seqs: list[str] (upper-case IUPAC) or a Reads; quals: numeric qualities (list of arrays or one concatenated uint8 array);
    rev: (seqs, quals) of the reverse mates, or None.  Options take one value or (forward, reverse).
    -> dict(seqs, quals[, rev_seqs, rev_quals]: the survivors in derep_reads' input form, reason: uint8[nreads] (0 kept, else
    the index in REASONS of the first stage that removed the read), flags: uint8[nreads] (MATE1 / MATE2 failed it, FLIPPED),
    src: int32[nout] input index of each survivor, stats)."""
    fwd = _as_reads(seqs, quals)
    rv = _as_reads(*rev) if rev is not None else None
    o = _opts(rv is not None, truncQ, truncLen, trimLeft, trimRight, maxLen, minLen, maxN, minQ, maxEE, rm_phix, rm_lowcomplex, orient_fwd,
              phix, n)
    r = _run(fwd, rv, o, device)
    out = {"reason": r["reason"], "flags": r["flags"], "src": r["src"], "stats": r["stats"], "reads": r["mates"],
           "seqs": r["mates"][0].strings(), "quals": r["mates"][0].qual}
    if rv is not None:
        out["rev_seqs"], out["rev_quals"] = r["mates"][1].strings(), r["mates"][1].qual
    return out


def test_filter_stages(seqs, quals, truncQ=2, truncLen=0, trimLeft=0, trimRight=0, maxLen=math.inf, minLen=20, maxN=0, minQ=0,
                       maxEE=math.inf, rm_phix=False, rm_lowcomplex=0, orient_fwd=None, phix=None, n=1e5, device=0):
    """Stage hook: the product's per-stage values for every read of one mate (STAGE_DTYPE), from dada2b_filter's own
    launch sequence.  phiX hits are computed when phix is given, complexity always."""
    rd = _as_reads(seqs, quals)
    o = _opts(False, truncQ, truncLen, trimLeft, trimRight, maxLen, minLen, maxN, minQ, maxEE, rm_phix, rm_lowcomplex, orient_fwd, phix, n)
    out = np.zeros(max(len(rd), 1), STAGE_DTYPE)
    eb = C.create_string_buffer(ERRLEN)
    ri = rd.c_in()
    rc = _lib().dada2b_test_filter_stages(C.byref(ri), C.byref(o), int(device), out.ctypes.data, eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    return out[:len(rd)]


test_filter_stages.__test__ = False


# ---- isPhiX / seqComplexity / C_matchRef -------------------------------------------------------------------------------
def C_matchRef(seqs, ref, word_size, non_overlapping, device=0):
    """src/filter.cpp:7-32 -> int32[nseq] hit counts."""
    seqs, buf, off = _pack_any(seqs)
    hits = np.zeros(max(len(seqs), 1), np.int32)
    eb = C.create_string_buffer(ERRLEN)
    rc = _lib().dada2b_match_ref(len(seqs), buf, off.ctypes.data, str(ref).encode(), int(word_size), int(bool(non_overlapping)), int(device),
                                 hits.ctypes.data, eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    return hits[:len(seqs)]


def _rc(s):
    return s[::-1].translate(str.maketrans("ACGTRYKMBVDHSWN", "TGCAYRMKVBHDSWN"))


def isPhiX(seqs, phix, wordSize=16, minMatches=2, nonOverlapping=True, device=0):
    """R/filter.R:1180-1187; phix: a FASTA path or the genome sequence.  -> bool[nseq]"""
    ph = _phix_seq(phix)
    hits = C_matchRef(seqs, ph, wordSize, nonOverlapping, device)
    hits_rc = C_matchRef(seqs, _rc(ph), wordSize, nonOverlapping, device)
    return (hits >= minMatches) | (hits_rc >= minMatches)


def seqComplexity(seqs, kmerSize=2, window=None, by=5, device=0):
    """R/filter.R:1248-1268 without window -> float64[nseq]; NaN where R gives NA (no A/C/G/T k-mer)."""
    if window is not None:
        raise api.Dada2bError("dada2b: seqComplexity with a window is not supported (only the whole-sequence form).")
    seqs, buf, off = _pack_any(seqs)
    if any(c not in IUPAC for c in set(buf.decode("latin-1"))):
        raise api.Dada2bError("dada2b: seqComplexity needs upper-case IUPAC DNA letters.")
    out = np.zeros(max(len(seqs), 1), np.float64)
    eb = C.create_string_buffer(ERRLEN)
    rc = _lib().dada2b_seq_complexity(len(seqs), buf, off.ctypes.data, int(kmerSize), 0, int(device), out.ctypes.data, eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    return out[:len(seqs)]


# ---- fastq ------------------------------------------------------------------------------------------------------------
def read_fastq_records(path, phred=33):
    """Four-line fastq(.gz) -> (ids list[bytes], Reads).  Letters must be upper-case IUPAC (checked on the device);
    qualities Phred+33 with the checks of derep.read_fastq."""
    op = gzip.open if str(path).endswith(".gz") else open
    with op(path, "rb") as f:
        data = f.read()
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()
    if len(lines) % 4:
        raise api.Dada2bError("dada2b: %s is not a four-line fastq file." % path)
    heads, seqs, plus, quals = lines[0::4], lines[1::4], lines[2::4], lines[3::4]
    if any(not h.startswith(b"@") for h in heads) or any(not p.startswith(b"+") for p in plus):
        raise api.Dada2bError("dada2b: %s is not a four-line fastq file." % path)
    lens = np.fromiter(map(len, seqs), dtype=np.int64, count=len(seqs))
    if not np.array_equal(lens, np.fromiter(map(len, quals), dtype=np.int64, count=len(quals))):
        raise api.Dada2bError("dada2b: sequence and quality lengths differ in %s." % path)
    off = np.zeros(len(seqs) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    qv = np.frombuffer(b"".join(quals), dtype=np.uint8).astype(np.int16) - phred
    if len(qv) and (qv.min() < 0 or qv.max() > 93):        # a wrong offset (e.g. Phred+64 data) must not wrap silently
        raise api.Dada2bError("dada2b: quality characters outside Phred+%d (0..93); only this encoding is supported "
                              "(the reference's qualityType = 'Auto' detection is not restated)." % phred)
    return [h[1:] for h in heads], Reads(b"".join(seqs), off, qv.astype(np.uint8))


def fastq_bytes(ids, reads, phred=33):
    """writeFastq's records: @id / sequence / + / quality, one per line."""
    s, q, o = reads.seq, (reads.qual + phred).astype(np.uint8).tobytes(), reads.off
    return b"".join(b"@%s\n%s\n+\n%s\n" % (ids[i], s[o[i]:o[i + 1]], q[o[i]:o[i + 1]]) for i in range(len(reads)))


def _write(path, data, compress):
    if compress:
        with open(path, "wb") as raw, gzip.GzipFile(filename="", mode="wb", fileobj=raw, mtime=0) as f:
            f.write(data)
    else:
        with open(path, "wb") as f:
            f.write(data)


def _check_common(matchIDs, multithread, qualityType):
    if matchIDs:
        raise api.Dada2bError("dada2b: matchIDs=True is not supported; reads must be in the same order in both files.")
    if multithread:
        raise api.Dada2bError("dada2b: multithread is not supported: the filter runs on the GPU.")
    if qualityType not in ("Auto", "FastqQuality"):
        raise api.Dada2bError("dada2b: only Phred+33 qualities are supported (qualityType 'Auto' is read as Phred+33).")


def _remove(path):
    if os.path.exists(path):
        os.remove(path)


def fastqFilter(fn, fout, truncQ=2, truncLen=0, maxLen=math.inf, minLen=20, trimLeft=0, trimRight=0, maxN=0, minQ=0, maxEE=math.inf,
                rm_phix=True, rm_lowcomplex=0, orient_fwd=None, n=1e6, OMP=True, qualityType="Auto", compress=True, verbose=False,
                phix=None, device=0):
    """R/filter.R:613-730 -> (reads.in, reads.out).  The output file is not written when no read survives."""
    _check_common(False, False, qualityType)
    for v in (truncQ, truncLen, maxLen, minLen, trimLeft, trimRight, maxN, minQ, maxEE):
        if isinstance(v, (list, tuple, np.ndarray)) and len(v) > 1:
            raise api.Dada2bError("Filtering and trimming arguments should be of length 1 when processing single-end (rather than "
                                  "paired-end) data.")
    if os.path.abspath(fn) == os.path.abspath(fout):
        raise api.Dada2bError("The output and input files must be different.")
    ids, reads = read_fastq_records(fn)
    _remove(fout)
    r = filter_reads(reads, None, None, truncQ, truncLen, trimLeft, trimRight, maxLen, minLen, maxN, minQ, maxEE, rm_phix, rm_lowcomplex,
                     orient_fwd, phix, n, device)
    nout = len(r["src"])
    if nout:
        _write(fout, fastq_bytes([ids[i] for i in r["src"]], r["reads"][0]), compress)
    if verbose:
        print("Read in %d, output %d (%.1f%%) filtered sequences." % (len(reads), nout, 100.0 * nout / max(len(reads), 1)))
    return len(reads), nout


def fastqPairedFilter(fn, fout, maxN=(0, 0), truncQ=(2, 2), truncLen=(0, 0), maxLen=(math.inf, math.inf), minLen=(20, 20), trimLeft=(0, 0),
                      trimRight=(0, 0), minQ=(0, 0), maxEE=(math.inf, math.inf), rm_phix=(True, True), rm_lowcomplex=(0, 0), matchIDs=False,
                      orient_fwd=None, id_sep=r"\s", id_field=None, n=1e6, OMP=True, qualityType="Auto", compress=True, verbose=False,
                      phix=None, device=0):
    """R/filter.R:878-1141.  fn, fout: (forward, reverse) paths -> (reads.in, reads.out)."""
    _check_common(matchIDs, False, qualityType)
    if len(fn) != 2:
        raise api.Dada2bError("Two paired input file names required.")
    if len(fout) != 2:
        raise api.Dada2bError("Two paired output file names required.")
    allp = [os.path.abspath(p) for p in list(fn) + list(fout)]
    if len(set(allp)) != 4:
        raise api.Dada2bError("The output and input file names must be different.")
    idsF, rdF = read_fastq_records(fn[0])
    idsR, rdR = read_fastq_records(fn[1])
    for p in fout:
        _remove(p)
    if len(rdF) != len(rdR):
        raise api.Dada2bError("Mismatched forward and reverse sequence files: %d, %d." % (len(rdF), len(rdR)))
    r = filter_reads(rdF, None, (rdR, None), truncQ, truncLen, trimLeft, trimRight, maxLen, minLen, maxN, minQ, maxEE, rm_phix,
                     rm_lowcomplex, orient_fwd, phix, n, device)
    src = r["src"]
    nout = len(src)
    if nout:
        sw = (r["flags"][src] & FLIPPED) != 0                # swapped pairs: the forward file gets the reverse read's id
        ids = (idsF, idsR)
        for m in range(2):
            rec_ids = [ids[1 - m if s else m][i] for i, s in zip(src, sw)]
            _write(fout[m], fastq_bytes(rec_ids, r["reads"][m]), compress)
    if verbose:
        print("Read in %d paired-sequences, output %d (%.1f%%) filtered paired-sequences." % (len(rdF), nout, 100.0 * nout / max(len(rdF), 1)))
    return len(rdF), nout


def _expand(files, outs):
    files = [files] if isinstance(files, (str, os.PathLike)) else list(files)
    if len(files) == 1 and os.path.isdir(files[0]):
        d = files[0]
        files = sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith((".fastq", ".fq", ".fastq.gz", ".fq.gz")))
    outs = [outs] if isinstance(outs, (str, os.PathLike)) else list(outs)
    if len(outs) == 1 and len(files) > 1:
        outs = [os.path.join(outs[0], os.path.basename(f)) for f in files]
    return files, outs


def filterAndTrim(fwd, filt, rev=None, filt_rev=None, compress=True, truncQ=2, truncLen=0, trimLeft=0, trimRight=0, maxLen=math.inf,
                  minLen=20, maxN=0, minQ=0, maxEE=math.inf, rm_phix=True, rm_lowcomplex=0, orient_fwd=None, matchIDs=False, id_sep=r"\s",
                  id_field=None, multithread=False, n=1e5, OMP=True, qualityType="Auto", verbose=False, phix=None, device=0):
    """R/filter.R:402-497 -> int64 [files x 2] matrix of (reads.in, reads.out), one row per input file in order.
    phix: a FASTA path or the phiX genome, required with rm_phix."""
    _check_common(matchIDs, multithread, qualityType)
    fwd, filt = _expand(fwd, filt)
    if not all(os.path.exists(f) for f in fwd):
        raise api.Dada2bError("Some input files do not exist.")
    if len(fwd) != len(filt):
        raise api.Dada2bError("Every input file must have a corresponding output file.")
    paired = rev is not None
    if paired:
        if filt_rev is None:
            raise api.Dada2bError("Output files for the reverse reads are required.")
        rev, filt_rev = _expand(rev, filt_rev)
        if not all(os.path.exists(f) for f in rev):
            raise api.Dada2bError("Some input files (rev) do not exist.")
        if len(rev) != len(fwd):
            raise api.Dada2bError("Paired forward and reverse input files must correspond.")
        if len(rev) != len(filt_rev):
            raise api.Dada2bError("Every input file (rev) must have a corresponding output file (filt.rev).")
    outs = [os.path.abspath(p) for p in filt + (filt_rev or [])]
    ins = [os.path.abspath(p) for p in fwd + (rev or [])]
    if len(set(outs)) != len(outs):
        raise api.Dada2bError("All output files must be distinct.")
    if set(outs) & set(ins):
        raise api.Dada2bError("Output files must be distinct from the input files.")
    for p in outs:
        os.makedirs(os.path.dirname(p), exist_ok=True)
    ph = _phix_seq(phix)
    rows = []
    for k in range(len(fwd)):
        if paired:
            rows.append(fastqPairedFilter((fwd[k], rev[k]), (filt[k], filt_rev[k]), maxN=maxN, truncQ=truncQ, truncLen=truncLen, maxLen=maxLen,
                                          minLen=minLen, trimLeft=trimLeft, trimRight=trimRight, minQ=minQ, maxEE=maxEE, rm_phix=rm_phix,
                                          rm_lowcomplex=rm_lowcomplex, orient_fwd=orient_fwd, n=n, qualityType=qualityType,
                                          compress=compress, verbose=verbose, phix=ph, device=device))
        else:
            rows.append(fastqFilter(fwd[k], filt[k], truncQ=truncQ, truncLen=truncLen, maxLen=maxLen, minLen=minLen, trimLeft=trimLeft,
                                    trimRight=trimRight, maxN=maxN, minQ=minQ, maxEE=maxEE, rm_phix=rm_phix, rm_lowcomplex=rm_lowcomplex,
                                    orient_fwd=orient_fwd, n=n, qualityType=qualityType, compress=compress, verbose=verbose, phix=ph,
                                    device=device))
    return np.array(rows, dtype=np.int64).reshape(len(fwd), 2)

"""Read quality checks for the GPU path: plotQualityProfile and plotComplexity (R/plot-methods.R:163-243, :293-309) up to
their ggplot calls.  No plot is drawn: each function returns the data frames R hands to ggplot, as dicts of columns.

The per-cycle quality table (ShortRead's qa(f, n)$perCycle$quality) is tallied in libdada2b.so behind
include/dada2b_qprofile.h, one call per file; complexities come from seqComplexity's device entry.  Fastq parsing, read
sampling and the per-cycle summaries run on the host.  No CPU fallback.

ShortRead's source is not part of the reference, so two of its results are read from their use in R/plot-methods.R:
  1. perCycle$quality has one row per (Cycle, Score) with Count > 0, and Score is the Phred score.
  2. readCounts$read is the number of reads qa tallied, i.e. min(reads in the file, n).
Cum and the labels are the same under either reading of (2).

Sampling: a file with at most n reads is used whole, and the output then equals R's.  Above n, R's FastqSampler draws n
reads with R's unseeded RNG, so R's own output changes from run to run.  Here one numpy.random.default_rng(seed) per call
draws, for each such file in order, n indices without replacement (rng.choice(nrec, n, replace=False), sorted); seed=None
is fresh entropy as in R, an int makes the draw reproducible.  n=None uses every read (an exact whole-file profile) and
acts as n = Inf.
"""
import ctypes as C
import math
import os

import numpy as np

from . import api
from . import filter as _flt
from .derep import DerepIn

NSCORE = 94
STATS = ("gpu_launches", "h2d_bytes", "d2h_bytes", "kernel_bytes", "ms_h2d", "ms_kernels", "ms_d2h", "ms_device", "ms_total")


class QProfileOut(C.Structure):
    _fields_ = [("ncycles", C.c_int32), ("counts", C.POINTER(C.c_int64)), ("nreads", C.c_int64), ("nbases", C.c_int64),
                ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64),
                ("ms_h2d", C.c_double), ("ms_kernels", C.c_double), ("ms_d2h", C.c_double), ("ms_device", C.c_double),
                ("ms_total", C.c_double)]


_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_quality_profile.argtypes = [P(DerepIn), C.c_int32, P(P(QProfileOut)), C.c_char_p]
        L.dada2b_qprofile_free.argtypes = [P(QProfileOut)]
        _BOUND = True
    return L


def quality_tally(off, qual, device=0):
    """dada2b_quality_profile on one read set: off int64[n+1] offsets into qual, qual uint8 numeric qualities.
    -> (counts int64[ncycles, 94], stats dict): counts[c, s] = number of bases with score s at 0-based cycle c."""
    off = np.ascontiguousarray(off, dtype=np.int64)
    qual = np.ascontiguousarray(qual, dtype=np.uint8)
    if len(off) < 1 or off[-1] > len(qual):
        raise api.Dada2bError("dada2b: offsets run past the qualities.")
    L = _lib()
    out = C.POINTER(QProfileOut)()
    eb = C.create_string_buffer(_flt.ERRLEN)
    ri = DerepIn(len(off) - 1, None, off.ctypes.data, qual.ctypes.data, 0)
    if L.dada2b_quality_profile(C.byref(ri), int(device), C.byref(out), eb):
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        nc = r.ncycles
        counts = np.ctypeslib.as_array(r.counts, shape=(max(nc * NSCORE, 1),))[:nc * NSCORE].reshape(nc, NSCORE).copy()
        stats = {s: getattr(r, s) for s in STATS}
        stats.update(nreads=r.nreads, nbases=r.nbases)
        return counts, stats
    finally:
        L.dada2b_qprofile_free(out)


# ---- files and sampling -----------------------------------------------------------------------------------------------
def _files(paths):
    if paths is None or isinstance(paths, (str, os.PathLike)):
        paths = [paths]
    return [f for f in paths if f is not None]                  # fl[!is.na(fl)]


def _check_n(n):
    if n is None or n == math.inf:
        return None
    if isinstance(n, bool) or not isinstance(n, (int, float, np.integer, np.floating)) or n != n or n != int(n) or n < 1:
        raise api.Dada2bError("dada2b: n must be a whole number >= 1, or None for every read (got %r)." % (n,))
    return int(n)


def _read(path):
    if not os.path.exists(path):
        raise api.Dada2bError("dada2b: the fastq file %s does not exist." % path)
    _, reads = _flt.read_fastq_records(path)
    if len(reads) == 0:
        raise api.Dada2bError("dada2b: the fastq file %s holds no reads." % path)
    return reads


def gather(reads, idx):
    """The reads idx (sorted int indices) of reads, as a new Reads; one np.repeat over the offsets, no loop per read."""
    lens = np.diff(reads.off)[idx]
    off = np.zeros(len(idx) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    pos = np.repeat(reads.off[idx] - off[:-1], lens) + np.arange(off[-1], dtype=np.int64)
    return _flt.Reads(np.frombuffer(reads.seq, np.uint8)[pos].tobytes(), off, reads.qual[pos])


def _sample(reads, n, rng):
    """The reads qa / FastqSampler sees: all of them up to n, else n drawn without replacement in file order."""
    if n is None or len(reads) <= n:
        return reads
    return gather(reads, np.sort(rng.choice(len(reads), n, replace=False)))


# ---- R's formatting and summaries -------------------------------------------------------------------------------------
def r_character(v):
    """as.character() of a whole-number double as R writes it: fixed notation unless scientific is narrower (ties go to
    fixed), e.g. 5e+05, 250000, 1e+05, 1000."""
    v = int(v)
    if v == 0:
        return "0"
    fixed = str(abs(v))
    digits = fixed.rstrip("0")
    sci = digits[0] + ("." + digits[1:] if len(digits) > 1 else "") + "e+%02d" % (len(fixed) - 1)
    return ("-" if v < 0 else "") + (fixed if len(fixed) <= len(sci) else sci)


def rclabel(rc, n):
    """paste("Reads >= ", n) when rc >= n, else paste("Reads: ", rc); rc is R's integer, n its double."""
    return "Reads >=  " + r_character(n) if n is not None and rc >= n else "Reads:  %d" % rc


def _stats(cycle, score, count, denom):
    """statdf's columns from rows (cycle, score, count) grouped by ascending cycle with ascending scores inside a cycle:
    rowsum means, get_quant at 0.25 / 0.5 / 0.75 and Cum = 10 * cums / denom, in float64 as R computes them."""
    cyc, start = np.unique(cycle, return_index=True)
    cums = np.add.reduceat(count, start) if len(cyc) else np.zeros(0, np.int64)
    sums = np.add.reduceat(score.astype(np.int64) * count, start) if len(cyc) else np.zeros(0, np.int64)
    quant = {0.25: [], 0.5: [], 0.75: []}
    for a, b, tot in zip(start, np.append(start[1:], len(cycle)), cums):
        frac = np.cumsum(count[a:b]).astype(np.float64) / np.float64(tot)
        for q, v in quant.items():
            v.append(score[a + int(np.argmax(frac >= q))])       # xx[which(cumsum(yy)/sum(yy) >= q)][[1]]
    return {"Cycle": cyc.astype(np.int32), "Mean": sums.astype(np.float64) / cums.astype(np.float64),
            "Q25": np.array(quant[0.25], np.int32), "Q50": np.array(quant[0.5], np.int32), "Q75": np.array(quant[0.75], np.int32),
            "Cum": 10.0 * cums.astype(np.float64) / np.float64(denom)}


def _concat(cols, types):
    return {k: (np.concatenate(v).astype(types[k]) if v else np.zeros(0, types[k])) if k in types else v for k, v in cols.items()}


TYPES = {"Cycle": np.int32, "Score": np.int32, "Count": np.int64, "Mean": np.float64, "Q25": np.int32, "Q50": np.int32, "Q75": np.int32,
         "Cum": np.float64}


def _aggregate(plotdf, nfiles, denom):
    """plotdf.summary (aggregate(Count ~ Cycle + Score, plotdf, sum): groups ordered by Score, then Cycle) and
    statdf.summary, with Cum over sum(pmin(rc, n)) = denom."""
    cyc, sc = plotdf["Cycle"].astype(np.int64), plotdf["Score"].astype(np.int64)
    span = int(cyc.max(initial=0)) + 1
    key, inv = np.unique(sc * span + cyc, return_inverse=True)
    count = np.zeros(len(key), np.int64)
    np.add.at(count, inv, plotdf["Count"])
    score, cycle = key // span, key % span
    label = "%d files (aggregated)" % nfiles
    pd = {"Cycle": cycle.astype(np.int32), "Score": score.astype(np.int32), "Count": count, "label": [label] * len(key)}
    o = np.lexsort((score, cycle))
    return pd, _stats(cycle[o], score[o].astype(np.int32), count[o], denom)


def plotQualityProfile(fl, n=500000, aggregate=False, seed=None, device=0):
    """plotQualityProfile (R/plot-methods.R:163-243) up to ggplot.  fl: a fastq(.gz) path or a list of them (None entries
    skipped), Phred+33.  n: reads per file (None: every read, as n = Inf); seed: the draw for files above n.  -> dict:
      plotdf  Cycle, Score, Count, file: one row per (file, cycle, score) with Count > 0 (Cycle 1-based), by file, cycle,
              score.  With aggregate, R's plotdf.summary: Cycle, Score, Count summed over files (int64), label; by score,
              then cycle.
      statdf  Cycle, Mean, Q25, Q50, Q75, Cum, file, one row per file and cycle; with aggregate, R's statdf.summary (no
              file column; Cum over sum(pmin(rc, n))).
      anndf   minScore (R replaces it by its minimum over the files), label, rclabel, rc, file: one row per file.
      nreads  int64: the records in each file.
    String columns are lists, the others numpy arrays.  A missing or empty file is an error.  The module docstring gives
    the sampling and the two readings of ShortRead's qa."""
    n = _check_n(n)
    files = _files(fl)
    rng = np.random.default_rng(seed)
    pd = {"Cycle": [], "Score": [], "Count": [], "file": []}
    sd = {k: [] for k in ("Cycle", "Mean", "Q25", "Q50", "Q75", "Cum", "file")}
    ann = {"minScore": [], "label": [], "rclabel": [], "rc": [], "file": []}
    nreads = []
    for f in files:
        reads = _read(f)
        nreads.append(len(reads))
        reads = _sample(reads, n, rng)
        rc = len(reads)                                        # readCounts$read: min(file reads, n)
        counts, _ = quality_tally(reads.off, reads.qual, device)
        name = os.path.basename(f)
        cyc, sc = np.nonzero(counts)                           # row-major: by cycle, then score
        cnt = counts[cyc, sc]
        cyc, sc = (cyc + 1).astype(np.int32), sc.astype(np.int32)
        pd["Cycle"].append(cyc); pd["Score"].append(sc); pd["Count"].append(cnt); pd["file"] += [name] * len(cyc)
        st = _stats(cyc, sc, cnt, rc)                          # min(rc, n) == rc
        for k, v in st.items():
            sd[k].append(v)
        sd["file"] += [name] * len(st["Cycle"])
        ann["minScore"].append(float(sc.min()) if len(sc) else np.inf)
        ann["label"].append(name)
        ann["rclabel"].append(rclabel(rc, n))
        ann["rc"].append(rc)
        ann["file"].append(name)
    pd, sd = _concat(pd, TYPES), _concat(sd, TYPES)
    ann["minScore"] = np.full(len(files), min(ann["minScore"], default=np.inf), np.float64)
    ann["rc"] = np.array(ann["rc"], np.int64)
    if aggregate:
        pd, sd = _aggregate(pd, len(files), int(ann["rc"].sum()))
    return {"plotdf": pd, "statdf": sd, "anndf": ann, "nreads": np.array(nreads, np.int64)}


def plotComplexity(fl, kmerSize=2, window=None, by=5, n=100000, aggregate=False, seed=None, device=0):
    """plotComplexity (R/plot-methods.R:293-309) up to ggplot.  fl: a fastq(.gz) path or a list of them (None entries
    skipped); each file sampled as in plotQualityProfile (n reads, default 1e5).  -> {"complexity": float64, "file":
    list}: seqComplexity of each file's sampled reads (in file order), files in order; NaN where R has NA.  With
    aggregate every label is "<k> files (aggregated)".  A window is refused as seqComplexity refuses it.  R's `bins`
    and `...` are ggplot's arguments and are not taken."""
    if window is not None:
        _flt.seqComplexity([], kmerSize, window, by, device)   # raises seqComplexity's refusal
    n = _check_n(n)
    files = _files(fl)
    rng = np.random.default_rng(seed)
    vals, names = [], []
    for f in files:
        reads = _sample(_read(f), n, rng)
        vals.append(_flt.seqComplexity(reads.strings(), kmerSize=kmerSize, device=device))
        names += [os.path.basename(f)] * len(reads)
    if aggregate:
        names = ["%d files (aggregated)" % len(files)] * len(names)
    return {"complexity": np.concatenate(vals) if vals else np.zeros(0), "file": names}

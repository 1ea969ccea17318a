"""Host-side mirror of the reference's dereplication for the GPU path (SURVEY.md 8(f1)).

`derep_reads` is what derepFastq() computes once ShortRead has parsed the fastq (qtables2 + the chunk loop,
/root/reference/R/sequenceIO.R:45-124, :150-183); `derepFastq` adds a plain fastq(.gz) reader for the tests.  All
computation happens in libdada2b.so behind include/dada2b_derep.h; this module only marshals.  No CPU fallback.
The result feeds dada2_b200.dada_uniques(uniques, abundances, None, err, quals) unchanged.
"""
import ctypes as C
import gzip

import numpy as np

from . import api

ERRLEN = 256


class DerepIn(C.Structure):
    _fields_ = [("nreads", C.c_int32), ("seq_concat", C.c_char_p), ("seq_off", C.c_void_p), ("qual_concat", C.c_void_p), ("chunk_n", C.c_int64)]


class DerepOut(C.Structure):
    _fields_ = [("nuniq", C.c_int32), ("maxlen", C.c_int32), ("nreads", C.c_int32), ("seq_concat", C.POINTER(C.c_char)),
                ("seq_off", C.POINTER(C.c_int64)), ("abund", C.POINTER(C.c_int32)), ("quals", C.POINTER(C.c_double)), ("map", C.POINTER(C.c_int32)),
                ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("ms_device", C.c_double), ("ms_sort", C.c_double), ("ms_total", C.c_double)]


class PoolIn(C.Structure):
    _fields_ = [("nsamples", C.c_int32), ("nuniq", C.c_void_p), ("maxlen", C.c_void_p), ("nmap", C.c_void_p), ("seq_concat", C.c_char_p),
                ("seq_off", C.c_void_p), ("abund", C.c_void_p), ("quals", C.c_void_p), ("map", C.c_void_p), ("prior", C.c_void_p)]


class PoolOut(C.Structure):
    _fields_ = [("npool", C.c_int32), ("maxlen", C.c_int32), ("nuniq_in", C.c_int64), ("nmap", C.c_int64),
                ("seq_concat", C.POINTER(C.c_char)), ("seq_off", C.POINTER(C.c_int64)), ("abund", C.POINTER(C.c_int32)),
                ("quals", C.POINTER(C.c_double)), ("map", C.POINTER(C.c_int32)), ("index", C.POINTER(C.c_int32)),
                ("prior", C.POINTER(C.c_uint8)), ("qmax", C.c_double), ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("ms_h2d", C.c_double), ("ms_kernels", C.c_double), ("ms_d2h", C.c_double), ("ms_total", C.c_double)]


POOL_STATS = ("gpu_launches", "h2d_bytes", "d2h_bytes", "ms_h2d", "ms_kernels", "ms_d2h", "ms_total")

_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_derep.argtypes = [P(DerepIn), C.c_int32, P(P(DerepOut)), C.c_char_p]
        L.dada2b_derep_free.argtypes = [P(DerepOut)]
        L.dada2b_derep_resident.argtypes = [P(DerepIn), C.c_int32, C.c_int32, P(P(DerepOut)), P(C.c_void_p), C.c_char_p]
        L.dada2b_pool.argtypes = [P(PoolIn), C.c_int32, C.c_int32, P(P(PoolOut)), C.c_char_p]
        L.dada2b_pool_resident.argtypes = [P(PoolIn), C.c_int32, C.c_int32, P(P(PoolOut)), P(C.c_void_p), C.c_char_p]
        L.dada2b_pool_free.argtypes = [P(PoolOut)]
        _BOUND = True
    return L


def derep_reads(seqs, quals, n=1000000, device=0, return_stats=False, resident=False, want_quals=True):
    """seqs: list[str] (A/C/G/T); quals: list of integer arrays or one uint8 array of all bases concatenated (numeric
    quality, Phred offset removed).  -> dict(uniques list[str], abundances int32[nuniq], quals float64[nuniq, maxlen]
    NaN/NA-padded, map int32[nreads] 1-based with NA = INT32_MIN) in derepFastq's order.
    resident=True: additionally leaves the uniques packed on the device and returns (dict, dada2_b200.Resident) -- run(err) on
    it is dada() on the dereplicated reads without the quality means ever visiting the host (want_quals=False drops them from
    the dict as well)."""
    L = _lib()
    nreads = len(seqs)
    lens = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=nreads)
    off = np.zeros(nreads + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    buf = "".join(seqs).encode()
    if isinstance(quals, np.ndarray) and quals.ndim == 1:
        q = np.ascontiguousarray(quals, dtype=np.uint8)
    else:
        q = np.ascontiguousarray(np.concatenate([np.asarray(x, dtype=np.uint8).ravel()[:l] for x, l in zip(quals, lens)]) if nreads else np.zeros(0, np.uint8))
    if len(q) != off[-1]:
        raise api.Dada2bError("dada2b: qualities and sequences have different lengths.")
    inp = DerepIn(nreads, buf, off.ctypes.data, q.ctypes.data, int(n))
    out = C.POINTER(DerepOut)()
    eb = C.create_string_buffer(ERRLEN)
    ctx = C.c_void_p()
    if resident:
        rc = L.dada2b_derep_resident(C.byref(inp), int(device), int(bool(want_quals)), C.byref(out), C.byref(ctx), eb)
    else:
        rc = L.dada2b_derep(C.byref(inp), int(device), C.byref(out), eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        nu, ml = r.nuniq, r.maxlen
        so = np.ctypeslib.as_array(r.seq_off, shape=(nu + 1,)).copy()
        raw = C.string_at(r.seq_concat, int(so[-1])).decode()
        res = {"uniques": [raw[so[i]:so[i + 1]] for i in range(nu)],
               "abundances": np.ctypeslib.as_array(r.abund, shape=(nu,)).copy(),
               "quals": np.ctypeslib.as_array(r.quals, shape=(nu, ml)).copy() if r.quals else None,   # maxlen x nuniq column-major == [nuniq, maxlen] row-major
               "map": np.ctypeslib.as_array(r.map, shape=(max(r.nreads, 1),))[:r.nreads].copy()}
        if return_stats:
            res["stats"] = {k: getattr(r, k) for k in ("gpu_launches", "h2d_bytes", "d2h_bytes", "ms_device", "ms_sort", "ms_total")}
        if resident:
            rs = api.Resident.__new__(api.Resident)                 # adopt the context the library built on the device
            rs._pin = None
            rs._ctx = ctx
            return res, rs
        return res
    finally:
        L.dada2b_derep_free(out)


def read_fastq(path, phred=33):
    """Plain four-line fastq(.gz) reader (host side; the reference uses ShortRead's FastqStreamer here)."""
    op = gzip.open if str(path).endswith(".gz") else open
    seqs, quals = [], []
    with op(path, "rt") as f:
        while True:
            if not f.readline():
                break
            s = f.readline().strip()
            f.readline()
            q = f.readline().strip()
            seqs.append(s)
            qv = np.frombuffer(q.encode(), dtype=np.uint8).astype(np.int16) - phred
            if len(qv) and (qv.min() < 0 or qv.max() > 93):        # a wrong offset (e.g. Phred+64 data) must not wrap silently
                raise api.Dada2bError("dada2b: quality characters outside Phred+%d (0..93); only this encoding is supported "
                                      "(the reference's qualityType = 'Auto' detection is not restated)." % phred)
            if len(s) and any(c not in "ACGT" for c in s):
                raise api.Dada2bError("dada2b: reads must be A/C/G/T (filter with maxN = 0 first, as the dada2 workflow does).")
            quals.append(qv.astype(np.uint8))
    return seqs, quals


def derepFastq(path, n=1000000, device=0):
    """derepFastq(fl, n) (R/sequenceIO.R:45) for one file: host fastq parsing + dada2b_derep."""
    seqs, quals = read_fastq(path)
    return derep_reads(seqs, quals, n=n, device=device)


def combineDereps2(dereps):
    """combineDereps2 (R/multiSample.R:165-203), the front door of dada(pool = TRUE): a list of derep results (dicts as
    returned by derep_reads / derepFastq) -> ONE derep whose uniques are the union in first-seen order, re-ordered by
    decreasing pooled abundance (stable, like order(decreasing = TRUE)); quality means pooled with the abundances as
    weights; the maps of the inputs concatenated and translated.  Host side, like the reference (it concatenates tables)."""
    if isinstance(dereps, dict):
        dereps = [dereps]
    maxlen = max(d["quals"].shape[1] for d in dereps)
    index = {}
    for d in dereps:                                        # unique(do.call(c, lapply(dereps, getSequences))): first occurrence order
        for s in d["uniques"]:
            if s not in index:
                index[s] = len(index)
    n = len(index)
    counts = np.zeros(n, dtype=np.int64)
    quals = np.zeros((n, maxlen), dtype=np.float64)
    maps = []
    for d in dereps:
        q = np.asarray(d["quals"], dtype=np.float64)
        if q.shape[1] < maxlen:
            q = np.concatenate([q, np.full((q.shape[0], maxlen - q.shape[1]), np.nan)], axis=1)
        ab = np.asarray(d["abundances"], dtype=np.int64)
        idx = np.fromiter((index[s] for s in d["uniques"]), dtype=np.int64, count=len(d["uniques"]))
        np.add.at(counts, idx, ab)
        np.add.at(quals, idx, q * ab[:, None])              # sweep(derep$quals, 1, derep$uniques, "*"): NA positions make the pooled mean NA, as in R
        m = np.asarray(d["map"], dtype=np.int64)
        maps.append(idx[m - 1] + 1)                         # map[derep$map], 1-based
    quals = quals / counts[:, None]
    order = np.argsort(-counts, kind="stable")              # order(derepCounts, decreasing = TRUE) keeps ties in input order
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.arange(n)
    seqs = list(index)
    newmap = rank[np.concatenate(maps) - 1] + 1 if maps else np.zeros(0, np.int64)
    return {"uniques": [seqs[i] for i in order], "abundances": counts[order].astype(np.int32), "quals": quals[order],
            "map": newmap.astype(np.int32)}


def pool_dereps(dereps, want_quals=True, device=0, priors=None, resident=False, return_stats=False):
    """combineDereps2 (R/multiSample.R:165-203) on the device (include/dada2b_pool.h): a list of derep dicts -> one derep
    dict (uniques, abundances, quals [npool, maxlen] or None without want_quals, map) equal to combineDereps2's, plus
    `index` (int32 per sample-unique, concatenated sample by sample: 1-based pooled position, match(names(derep_s$uniques),
    names(pooled))), `qmax` (largest non-NA pooled mean) and `prior` (bool per pooled unique: OR of `priors`, one bool array per sample, over the occurrences).
    resident=True: additionally leaves the pooled uniques packed on the device with their prior flags and returns
    (dict, dada2_b200.Resident); run(err) on it is dada() on the pooled derep."""
    if isinstance(dereps, dict):
        dereps = [dereps]
    L = _lib()
    S = len(dereps)
    seqs = [u for d in dereps for u in d["uniques"]]
    nuniq = np.array([len(d["uniques"]) for d in dereps], np.int32)
    qs = [np.asarray(d["quals"], dtype=np.float64) for d in dereps]
    for d, q in zip(dereps, qs):
        if q.ndim != 2 or q.shape[0] != len(d["uniques"]):
            raise api.Dada2bError("derep$quals matrices must have one row for each derep$unique sequence.")
    maxlen = np.array([q.shape[1] for q in qs], np.int32)
    maps = [np.asarray(d["map"], dtype=np.int32).ravel() for d in dereps]
    nmap = np.array([len(m) for m in maps], np.int64)
    lens = np.fromiter((len(x) for x in seqs), dtype=np.int64, count=len(seqs))
    off = np.zeros(len(seqs) + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    buf = "".join(seqs).encode()
    ab = np.ascontiguousarray(np.concatenate([np.asarray(d["abundances"]) for d in dereps]) if S else np.zeros(0), dtype=np.int32)
    if len(ab) != len(seqs):
        raise api.Dada2bError("derep$uniques and its abundances have different lengths.")
    qcat = np.ascontiguousarray(np.concatenate([q.ravel() for q in qs]) if S else np.zeros(0))
    mcat = np.ascontiguousarray(np.concatenate(maps) if S else np.zeros(0, np.int32))
    pr = None
    if priors is not None:
        pr = np.ascontiguousarray(np.concatenate([np.asarray(p, dtype=bool).ravel() for p in priors]), dtype=np.uint8)
        if len(pr) != len(seqs):
            raise api.Dada2bError("Sequence and priors vectors had different lengths.")
    inp = PoolIn(S, nuniq.ctypes.data, maxlen.ctypes.data, nmap.ctypes.data, buf, off.ctypes.data, ab.ctypes.data, qcat.ctypes.data,
                 mcat.ctypes.data, pr.ctypes.data if pr is not None else None)
    out = C.POINTER(PoolOut)()
    eb = C.create_string_buffer(ERRLEN)
    ctx = C.c_void_p()
    if resident:
        rc = L.dada2b_pool_resident(C.byref(inp), int(device), int(bool(want_quals)), C.byref(out), C.byref(ctx), eb)
    else:
        rc = L.dada2b_pool(C.byref(inp), int(device), int(bool(want_quals)), C.byref(out), eb)
    if rc:
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        nu, ml = r.npool, r.maxlen
        so = np.ctypeslib.as_array(r.seq_off, shape=(nu + 1,)).copy()
        raw = C.string_at(r.seq_concat, int(so[-1])).decode()
        res = {"uniques": [raw[so[i]:so[i + 1]] for i in range(nu)],
               "abundances": np.ctypeslib.as_array(r.abund, shape=(nu,)).copy(),
               "quals": np.ctypeslib.as_array(r.quals, shape=(nu, ml)).copy() if r.quals else None,
               "map": np.ctypeslib.as_array(r.map, shape=(max(r.nmap, 1),))[:r.nmap].copy(),
               "index": np.ctypeslib.as_array(r.index, shape=(r.nuniq_in,)).copy(),
               "prior": np.ctypeslib.as_array(r.prior, shape=(nu,)).astype(bool), "qmax": r.qmax}
        if return_stats:
            res["stats"] = {k: getattr(r, k) for k in POOL_STATS}
        if resident:
            rs = api.Resident.__new__(api.Resident)                 # adopt the context the library built on the device
            rs._pin = None
            rs._ctx = ctx
            rs.nraw = nu
            return res, rs
        return res
    finally:
        L.dada2b_pool_free(out)

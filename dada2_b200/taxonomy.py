"""Taxonomic classification on the GPU: assignTaxonomy (R/taxonomy.R:65-160) and C_assign_taxonomy2.

The naive Bayesian classifier (8-mer table, main assignment, 100 bootstraps) runs in libdada2b.so behind
include/dada2b_taxonomy.h; this module parses the training fasta, restates the R wrapper around the native call and
marshals.  `TaxDB` keeps one table resident on the device for any number of `classify` calls.  No CPU fallback.
"""
import ctypes as C
import gzip
import os
import re
import warnings

import numpy as np

from . import api

ERRLEN = 256
NBOOT = 100
MIN_REF_LEN = 20
MIN_TAX_LEN = 50
NA = -(2 ** 31)
UNSPEC = "_DADA2_UNSPECIFIED"
TAX_LEVELS = ("Kingdom", "Phylum", "Class", "Order", "Family", "Genus", "Species")


class TaxOpts(C.Structure):
    _fields_ = [("max_table_bytes", C.c_int64), ("chunk_genera", C.c_int32), ("reserved", C.c_int32)]


class TaxSeqs(C.Structure):
    _fields_ = [("n", C.c_int32), ("reserved", C.c_int32), ("seq_concat", C.c_char_p), ("seq_off", C.POINTER(C.c_int64))]


class TaxDBInfo(C.Structure):
    _fields_ = [("nref", C.c_int32), ("ngenus", C.c_int32), ("nlevel", C.c_int32), ("nchunk", C.c_int32), ("chunk_genera", C.c_int32),
                ("reserved", C.c_int32), ("table_bytes", C.c_int64), ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64),
                ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64), ("ms_h2d", C.c_double), ("ms_kernels", C.c_double),
                ("ms_d2h", C.c_double), ("ms_device", C.c_double), ("ms_total", C.c_double)]


class TaxOut(C.Structure):
    _fields_ = [("nseq", C.c_int32), ("nlevel", C.c_int32), ("tax", C.POINTER(C.c_int32)), ("boot", C.POINTER(C.c_int32)),
                ("boot_tax", C.POINTER(C.c_int32)), ("logp", C.POINTER(C.c_float)), ("used_rc", C.POINTER(C.c_uint8)),
                ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64),
                ("ms_h2d", C.c_double), ("ms_kernels", C.c_double), ("ms_d2h", C.c_double), ("ms_device", C.c_double),
                ("ms_total", C.c_double)]


STATS = ("gpu_launches", "h2d_bytes", "d2h_bytes", "kernel_bytes", "ms_h2d", "ms_kernels", "ms_d2h", "ms_device", "ms_total")

_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_tax_default_opts.argtypes = [P(TaxOpts)]
        L.dada2b_tax_db_build.argtypes = [P(TaxSeqs), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, P(TaxOpts), C.c_int32, P(C.c_void_p),
                                          C.c_char_p]
        L.dada2b_tax_db_info_get.argtypes = [C.c_void_p, P(TaxDBInfo)]
        L.dada2b_tax_db_free.argtypes = [C.c_void_p]
        L.dada2b_tax_classify.argtypes = [C.c_void_p, P(TaxSeqs), C.c_int32, C.c_void_p, C.c_int64, C.c_uint64, P(P(TaxOut)), C.c_char_p]
        L.dada2b_tax_free.argtypes = [P(TaxOut)]
        L.dada2b_assign_taxonomy.argtypes = [P(TaxSeqs), P(TaxSeqs), C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_int64, C.c_uint64, C.c_int32, P(P(TaxOut)), C.c_char_p]
        L.dada2b_test_tax_table.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_char_p]
        L.dada2b_test_tax_logp.argtypes = [C.c_void_p, P(TaxSeqs), C.c_void_p, C.c_char_p]
        _BOUND = True
    return L


class _Seqs:
    """Strings (str or bytes) concatenated for the C-ABI; keeps the buffers alive."""

    def __init__(self, seqs):
        bs = [s.encode() if isinstance(s, str) else bytes(s) for s in seqs]
        self.off = np.zeros(len(bs) + 1, np.int64)
        np.cumsum([len(b) for b in bs], out=self.off[1:])
        self.buf = b"".join(bs) or b"\0"
        self.c = TaxSeqs(len(bs), 0, self.buf, self.off.ctypes.data_as(C.POINTER(C.c_int64)))


def _seed(seed):
    return int.from_bytes(os.urandom(8), "little") if seed is None else int(seed) & (2 ** 64 - 1)


def _unifs(unifs):
    if unifs is None:
        return None, 0
    u = np.ascontiguousarray(unifs, dtype=np.float64)
    return u, u.size


def _out(p):
    r = p.contents
    n, nl = r.nseq, r.nlevel
    arr = np.ctypeslib.as_array
    return {"tax": arr(r.tax, shape=(n,)).copy(), "boot": arr(r.boot, shape=(n * nl,)).reshape(n, nl).copy(),
            "boot_tax": arr(r.boot_tax, shape=(n * NBOOT,)).reshape(n, NBOOT).copy(), "logp": arr(r.logp, shape=(n,)).copy(),
            "used_rc": arr(r.used_rc, shape=(n,)).astype(bool), "stats": {s: getattr(r, s) for s in STATS}}


def _classify_call(fn, *args):
    out = C.POINTER(TaxOut)()
    eb = C.create_string_buffer(ERRLEN)
    if fn(*args, C.byref(out), eb):
        raise api.Dada2bError(eb.value.decode())
    try:
        return _out(out)
    finally:
        _lib().dada2b_tax_free(out)


def _genusmat(genusmat):
    gm = np.ascontiguousarray(genusmat, dtype=np.int32)
    if gm.ndim != 2:
        raise api.Dada2bError("genusmat must be a matrix.")
    return gm


def C_assign_taxonomy2(seqs, rcs, refs, ref_to_genus, genusmat, try_rc, verbose=False, unifs=None, seed=None, device=0):
    """src/taxonomy.cpp:206-338 -> dict(tax [nseq] 1-based genus or NA, boot [nseq, nlevel], boot_tax [nseq, 100], logp, used_rc,
    stats).  rcs is accepted for the reference's signature and ignored: the reverse complement's k-mers are derived from the
    forward ones.  unifs: the reference's runif buffer (nseq * 100 * (max_arraylen / 8) values); None draws from seed."""
    if len(seqs) == 0:
        raise api.Dada2bError("No seqs provided to classify.")
    if len(refs) != len(ref_to_genus):
        raise api.Dada2bError("Length mismatch between number of references and map to genus.")
    gm = _genusmat(genusmat)
    rg = np.ascontiguousarray(ref_to_genus, dtype=np.int32)
    q, r = _Seqs(seqs), _Seqs(refs)
    u, nu = _unifs(unifs)
    L = _lib()
    if verbose:
        print("Finished processing reference fasta.", end="")
    return _classify_call(L.dada2b_assign_taxonomy, C.byref(q.c), C.byref(r.c), rg.ctypes.data, gm.ctypes.data, gm.shape[0], gm.shape[1],
                          int(bool(try_rc)), None if u is None else u.ctypes.data, nu, _seed(seed), int(device))


# ---- the training fasta and R's wrapper rules ----
def read_fasta(path):
    """(ids, seqs) of a fasta file (gzip by magic bytes), as ShortRead's readFasta: the whole header line, sequence lines
    joined without whitespace and upper-cased (DNAStringSet)."""
    with open(path, "rb") as f:
        magic = f.read(2)
    op = gzip.open if magic == b"\x1f\x8b" else open
    ids, seqs, cur = [], [], []
    with op(path, "rb") as f:
        for line in f:
            line = line.rstrip(b"\r\n")
            if line.startswith(b">"):
                if ids:
                    seqs.append(b"".join(cur).upper().decode())
                ids.append(line[1:].decode())
                cur = []
            elif ids:
                cur.append(b"".join(line.split()))
    if ids:
        seqs.append(b"".join(cur).upper().decode())
    return ids, seqs


def _r_strsplit(s, sep):
    """strsplit(s, sep) with a literal one-letter sep: a trailing empty field is dropped."""
    parts = s.split(sep)
    if parts and parts[-1] == "":
        parts.pop()
    return parts


_WS = re.compile(r"\s", re.ASCII)


def parse_training(ids, refs):
    """R/taxonomy.R:76-122 after readFasta: -> (refs, genus_unq, ref_to_genus (1-based), genusmat [ngenus, td], td)."""
    lens = np.array([len(r) for r in refs], dtype=np.int64)
    if np.any(lens < MIN_REF_LEN):
        keep = lens >= MIN_REF_LEN
        refs = [r for r, k in zip(refs, keep) if k]
        ids = [t for t, k in zip(ids, keep) if k]
        warnings.warn("Some reference sequences were too short (<%dnts) and were excluded." % MIN_REF_LEN)
    if not refs:
        raise api.Dada2bError("dada2b: no reference sequence of at least %d nt." % MIN_REF_LEN)
    tax = [t.strip() for t in ids]
    if len(tax) >= 10 and all(re.search(r"FU\|re[pf]s", t) for t in tax[:10]):        # tax[1:10]: NA (not UNITE) below 10
        print("UNITE fungal taxonomic reference detected.")
        tax = [(t.split("|")[4] if len(t.split("|")) > 4 else "NA") for t in tax]
        tax = [re.sub(r"[pcofg]__unidentified;", UNSPEC + ";", t) for t in tax]
        tax = [re.sub(r";s__(\w+)_", ";s__", t, flags=re.ASCII) for t in tax]
        tax = [re.sub(r";s__sp$", ";" + UNSPEC, t) for t in tax]
    if ";" not in tax[0]:
        if len(_r_strsplit_ws(tax[0])) == 3:
            raise api.Dada2bError("Incorrect reference file format for assignTaxonomy (this looks like a file formatted for assignSpecies).")
        raise api.Dada2bError("Incorrect reference file format for assignTaxonomy.")
    depth = [len(_r_strsplit(t, ";")) for t in tax]
    td = max(depth)
    tax = [t + (UNSPEC + ";") * (td - d) for t, d in zip(tax, depth)]
    index = {}
    for t in tax:
        index.setdefault(t, len(index))
    genus_unq = list(index)
    ref_to_genus = np.array([index[t] + 1 for t in tax], dtype=np.int32)
    # matrix(unlist(strsplit(genus.unq, ";")), ncol=td, byrow=TRUE): fields flattened, rows filled in order, recycled
    flat = [f for g in genus_unq for f in _r_strsplit(g, ";")]
    nrow = -(-len(flat) // td)
    if len(flat) % td:
        warnings.warn("data length [%d] is not a sub-multiple or multiple of the number of columns [%d]" % (len(flat), td))
    cells = [flat[i % len(flat)] for i in range(nrow * td)]
    gm = np.zeros((nrow, td), np.int32)
    for lev in range(td):
        codes = {}
        for r in range(nrow):
            gm[r, lev] = codes.setdefault(cells[r * td + lev], len(codes) + 1)
    return refs, genus_unq, ref_to_genus, gm, td


def _r_strsplit_ws(s):
    parts = _WS.split(s)
    if parts and parts[-1] == "":
        parts.pop()
    return parts


def get_sequences(seqs):
    """getSequences for the inputs this package produces: strings, a makeSequenceTable result (its column names) or a
    dada result (its clustering's sequences)."""
    if isinstance(seqs, str):
        return [seqs]
    if isinstance(seqs, dict) and "clustering" in seqs:
        return list(seqs["clustering"]["sequence"])
    if isinstance(seqs, tuple) and len(seqs) == 3 and isinstance(seqs[0], np.ndarray):
        return list(seqs[1])
    return [s.decode() if isinstance(s, bytes) else str(s) for s in seqs]


def _assemble(res, seqs, genus_unq, td, minBoot, taxLevels, outputBootstraps):
    """R/taxonomy.R:136-159 -> object array [nseq, td] (None for NA) with the level names, or a dict with the boot matrix."""
    n = len(seqs)
    out = np.full((n, td), None, dtype=object)
    for i in range(n):
        t = res["tax"][i]
        if t == NA:
            continue                                       # genus.unq[NA]: the row stays NA at any minBoot
        lev = _r_strsplit(genus_unq[t - 1], ";")
        sel = [lev[k] if k < len(lev) else None for k in range(td) if res["boot"][i, k] >= minBoot]
        out[i, :len(sel)] = sel
    out[out == UNSPEC] = None
    names = [taxLevels[k] if k < len(taxLevels) else None for k in range(td)]
    if outputBootstraps:
        return {"tax": out, "boot": res["boot"].copy(), "levels": names, "seqs": list(seqs)}
    return out, names


class TaxDB:
    """A training set parsed once with its table resident on the device; classify() as often as needed.
    refFasta: a path, or (ids, seqs) of an already read fasta.  max_table_bytes / chunk_genera: see dada2b_tax_opts."""

    def __init__(self, refFasta, device=0, max_table_bytes=0, chunk_genera=0, verbose=False):
        ids, refs = read_fasta(refFasta) if isinstance(refFasta, (str, os.PathLike)) else refFasta
        refs, self.genus_unq, self.ref_to_genus, self.genusmat, self.td = parse_training(list(ids), list(refs))
        self._db = None
        self.device = int(device)
        self._build(refs, max_table_bytes, chunk_genera)
        if verbose:
            print("Finished processing reference fasta.")

    @classmethod
    def from_arrays(cls, refs, ref_to_genus, genusmat, device=0, max_table_bytes=0, chunk_genera=0):
        """The native database of C_assign_taxonomy2's inputs (no fasta, no wrapper rules)."""
        self = cls.__new__(cls)
        self._db = None
        self.device = int(device)
        self.genus_unq, self.ref_to_genus, self.genusmat = None, np.asarray(ref_to_genus, np.int32), _genusmat(genusmat)
        self.td = self.genusmat.shape[1]
        self._build(list(refs), max_table_bytes, chunk_genera)
        return self

    def _build(self, refs, max_table_bytes, chunk_genera):
        L = _lib()
        if len(refs) != len(self.ref_to_genus):
            raise api.Dada2bError("Length mismatch between number of references and map to genus.")
        o = TaxOpts()
        L.dada2b_tax_default_opts(C.byref(o))
        o.max_table_bytes, o.chunk_genera = int(max_table_bytes), int(chunk_genera)
        r = _Seqs(refs)
        rg = np.ascontiguousarray(self.ref_to_genus, np.int32)
        db = C.c_void_p()
        eb = C.create_string_buffer(ERRLEN)
        if L.dada2b_tax_db_build(C.byref(r.c), rg.ctypes.data, self.genusmat.ctypes.data, self.genusmat.shape[0], self.genusmat.shape[1],
                                 C.byref(o), self.device, C.byref(db), eb):
            raise api.Dada2bError(eb.value.decode())
        self._db = db
        info = TaxDBInfo()
        L.dada2b_tax_db_info_get(db, C.byref(info))
        self.info = {k: getattr(info, k) for k, _ in TaxDBInfo._fields_ if k != "reserved"}

    @property
    def ngenus(self):
        return self.genusmat.shape[0]

    def close(self):
        if self._db:
            _lib().dada2b_tax_db_free(self._db)
            self._db = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def raw(self, seqs, tryRC=False, unifs=None, seed=None):
        """The native classification (C_assign_taxonomy2's result) of a list of strings."""
        if not self._db:
            raise api.Dada2bError("dada2b: the database was closed.")
        q = _Seqs(seqs)
        u, nu = _unifs(unifs)
        return _classify_call(_lib().dada2b_tax_classify, self._db, C.byref(q.c), int(bool(tryRC)), None if u is None else u.ctypes.data,
                              nu, _seed(seed))

    def classify(self, seqs, minBoot=50, tryRC=False, outputBootstraps=False, taxLevels=TAX_LEVELS, seed=None, unifs=None):
        """assignTaxonomy's result for seqs against this database."""
        seqs = get_sequences(seqs)
        if self.genus_unq is None:
            raise api.Dada2bError("dada2b: a database built from arrays has no taxonomy strings; use raw().")
        if seqs and min(len(s) for s in seqs) < MIN_TAX_LEN:
            warnings.warn("Some sequences were shorter than %d nts and will not receive a taxonomic classification." % MIN_TAX_LEN)
        res = self.raw(seqs, tryRC, unifs, seed)
        return _assemble(res, seqs, self.genus_unq, self.td, minBoot, list(taxLevels), outputBootstraps)

    def table(self, kmers, genera):
        """Test hook: float32 [len(kmers), len(genera)] entries of the device table (0-based genera)."""
        k = np.ascontiguousarray(kmers, np.int32)
        g = np.ascontiguousarray(genera, np.int32)
        out = np.zeros((max(k.size, 1), max(g.size, 1)), np.float32)
        eb = C.create_string_buffer(ERRLEN)
        if _lib().dada2b_test_tax_table(self._db, k.size, k.ctypes.data, g.size, g.ctypes.data, out.ctypes.data, eb):
            raise api.Dada2bError(eb.value.decode())
        return out[:k.size, :g.size]

    def logp(self, seqs):
        """Test hook: float32 [nseq, 2, ngenus] forward and reverse-complement main logp of every query for every genus."""
        q = _Seqs(seqs)
        out = np.zeros((max(len(seqs), 1), 2, self.ngenus), np.float32)
        eb = C.create_string_buffer(ERRLEN)
        if _lib().dada2b_test_tax_logp(self._db, C.byref(q.c), out.ctypes.data, eb):
            raise api.Dada2bError(eb.value.decode())
        return out[:len(seqs)]


def assignTaxonomy(seqs, refFasta, minBoot=50, tryRC=False, outputBootstraps=False, taxLevels=TAX_LEVELS, multithread=False, verbose=False,
                   seed=None, device=0, unifs=None):
    """R/taxonomy.R:65-160.  -> (object array [nseq, td] with None for NA, level names), or with outputBootstraps a dict
    (tax, boot, levels, seqs).  multithread is accepted and ignored (the work is on the GPU).  seed: the draws and the tie
    rule (DESIGN.md 21); unifs: the reference's runif buffer instead of the seeded draws."""
    seqs = get_sequences(seqs)
    if seqs and min(len(s) for s in seqs) < MIN_TAX_LEN:
        warnings.warn("Some sequences were shorter than %d nts and will not receive a taxonomic classification." % MIN_TAX_LEN)
    db = TaxDB(refFasta, device=device, verbose=verbose)
    try:
        res = db.raw(seqs, tryRC, unifs, seed)
    finally:
        db.close()
    return _assemble(res, seqs, db.genus_unq, db.td, minBoot, list(taxLevels), outputBootstraps)

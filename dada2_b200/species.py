"""Species assignment by exact matching on the GPU: assignSpecies and addSpecies (R/taxonomy.R:162-360).

The exact substring search of every query in every reference of a species fasta (the PDict / vcountPDict loop of
assignSpecies) and the reduction of the hits to distinct genus and species labels run in libdada2b.so behind
include/dada2b_species.h.  This module parses the fasta, restates R's wrapper rules (the format check, the label
fields, mapHits, matchGenera, addSpecies' merge) and marshals.  `SpeciesDB` keeps the references resident on the device
for any number of calls.  No CPU fallback.

Pinned deviations from R (DESIGN.md 22): labels are sorted in byte order (R follows the session's collation); the
regular expressions of matchGenera are Python's `re` (R uses TRE); an empty query is refused (R's PDict fails on it);
`n` must be a positive integer.
"""
import ctypes as C
import os
import re

import numpy as np

from . import api
from .taxonomy import _r_strsplit_ws, get_sequences, read_fasta

ERRLEN = 256
LEVELS = ["Genus", "Species"]
ECOLI = "Escherichia/Shigella"


class SpeciesSeqs(C.Structure):
    _fields_ = [("n", C.c_int32), ("reserved", C.c_int32), ("seq_concat", C.c_char_p), ("seq_off", C.POINTER(C.c_int64))]


class SpeciesDBInfo(C.Structure):
    _fields_ = [("nref", C.c_int32), ("reserved", C.c_int32), ("nbases", C.c_int64), ("device_bytes", C.c_int64),
                ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64),
                ("ms_h2d", C.c_double), ("ms_kernels", C.c_double), ("ms_d2h", C.c_double), ("ms_device", C.c_double),
                ("ms_total", C.c_double)]


class SpeciesOut(C.Structure):
    _fields_ = [("nseq", C.c_int32), ("reserved", C.c_int32), ("nhits", C.POINTER(C.c_int32)), ("genus_n", C.POINTER(C.c_int32)),
                ("genus_off", C.POINTER(C.c_int64)), ("genus_ids", C.POINTER(C.c_int32)), ("species_n", C.POINTER(C.c_int32)),
                ("species_ids", C.POINTER(C.c_int32)), ("species_off", C.POINTER(C.c_int64)), ("hit_off", C.POINTER(C.c_int64)),
                ("hit_refs", C.POINTER(C.c_int32)), ("npatterns", C.c_int64), ("hit_records", C.c_int64), ("hit_capacity", C.c_int64),
                ("distinct_hits", C.c_int64), ("scans", C.c_int32), ("max_group", C.c_int32), ("gpu_launches", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("kernel_bytes", C.c_int64), ("ms_h2d", C.c_double),
                ("ms_scan", C.c_double), ("ms_reduce", C.c_double), ("ms_d2h", C.c_double), ("ms_device", C.c_double),
                ("ms_total", C.c_double)]


STATS = ("npatterns", "hit_records", "hit_capacity", "distinct_hits", "scans", "max_group", "gpu_launches", "h2d_bytes", "d2h_bytes",
         "kernel_bytes", "ms_h2d", "ms_scan", "ms_reduce", "ms_d2h", "ms_device", "ms_total")

_BOUND = False


def _lib():
    global _BOUND
    L = api.lib()
    if not _BOUND:
        P = C.POINTER
        L.dada2b_species_db_build.argtypes = [P(SpeciesSeqs), C.c_void_p, C.c_void_p, C.c_int32, P(C.c_void_p), C.c_char_p]
        L.dada2b_species_db_info_get.argtypes = [C.c_void_p, P(SpeciesDBInfo)]
        L.dada2b_species_db_free.argtypes = [C.c_void_p]
        L.dada2b_species_assign.argtypes = [C.c_void_p, P(SpeciesSeqs), C.c_int32, C.c_int32, C.c_int32, P(P(SpeciesOut)), C.c_char_p]
        L.dada2b_species_free.argtypes = [P(SpeciesOut)]
        L.dada2b_test_species_hits.argtypes = [C.c_void_p, P(SpeciesSeqs), C.c_int32, P(P(SpeciesOut)), C.c_char_p]
        _BOUND = True
    return L


class _Seqs:
    """Strings concatenated for the C-ABI; keeps the buffers alive."""

    def __init__(self, seqs):
        bs = [s.encode() if isinstance(s, str) else bytes(s) for s in seqs]
        self.off = np.zeros(len(bs) + 1, np.int64)
        np.cumsum([len(b) for b in bs], out=self.off[1:])
        self.buf = b"".join(bs) or b"\0"
        self.c = SpeciesSeqs(len(bs), 0, self.buf, self.off.ctypes.data_as(C.POINTER(C.c_int64)))


def _csr(n, off, ids, nseq):
    """Per query: the label-id list, or None where the list was cut (its count exceeded keep)."""
    arr = np.ctypeslib.as_array
    cnt = arr(n, shape=(nseq,)).copy()
    o = arr(off, shape=(nseq + 1,)).copy()
    v = arr(ids, shape=(max(int(o[-1]), 1),))[:int(o[-1])].copy()
    return cnt, [v[o[i]:o[i + 1]] if o[i + 1] - o[i] == cnt[i] else None for i in range(nseq)]


def _native(fn, *args, hits=False):
    out = C.POINTER(SpeciesOut)()
    eb = C.create_string_buffer(ERRLEN)
    if fn(*args, C.byref(out), eb):
        raise api.Dada2bError(eb.value.decode())
    try:
        r = out.contents
        n = r.nseq
        res = {"nhits": np.ctypeslib.as_array(r.nhits, shape=(n,)).copy() if n else np.zeros(0, np.int32),
               "stats": {s: getattr(r, s) for s in STATS}}
        if n:
            res["genus_n"], res["genus"] = _csr(r.genus_n, r.genus_off, r.genus_ids, n)
            res["species_n"], res["species"] = _csr(r.species_n, r.species_off, r.species_ids, n)
        else:
            res["genus_n"] = res["species_n"] = np.zeros(0, np.int32)
            res["genus"] = res["species"] = []
        if hits:
            o = np.ctypeslib.as_array(r.hit_off, shape=(n + 1,)).copy()
            v = np.ctypeslib.as_array(r.hit_refs, shape=(max(int(o[-1]), 1),))[:int(o[-1])].copy()
            res["hits"] = [v[o[i]:o[i + 1]] for i in range(n)]
        return res
    finally:
        _lib().dada2b_species_free(out)


# ---- R's wrapper rules ----
def keep_of(allowMultiple):
    """assignSpecies' keep: FALSE -> 1, TRUE -> Inf, otherwise as.integer(allowMultiple)."""
    if isinstance(allowMultiple, (bool, np.bool_)):
        return float("inf") if allowMultiple else 1
    return int(allowMultiple)


def parse_species(ids):
    """R/taxonomy.R:255-263: the format check on the first id, then genus = field 2 and species = field 3 of a split on
    single whitespace characters (None where a field is missing)."""
    if not ids:
        raise api.Dada2bError("dada2b: the reference fasta holds no sequences.")
    if not len(_r_strsplit_ws(ids[0])) >= 3:
        if ids[0].count(";") >= 3:
            raise api.Dada2bError("Incorrect reference file format for assignSpecies (this looks like a file formatted for assignTaxonomy).")
        raise api.Dada2bError("Incorrect reference file format for assignSpecies.")
    fields = [_r_strsplit_ws(t) for t in ids]
    genus = [f[1] if len(f) > 1 else None for f in fields]
    species = [f[2] if len(f) > 2 else None for f in fields]
    return genus, species


def relabel(label):
    """mapHits' first step: a label containing Escherichia or Shigella becomes Escherichia/Shigella."""
    if label is not None and ("Escherichia" in label or "Shigella" in label):
        return ECOLI
    return label


def label_ids(labels):
    """-> (int32 ids, 0 for NA; names with names[0] = None) of the relabelled labels, in order of first appearance."""
    index = {None: 0}
    ids = np.array([index.setdefault(relabel(t), len(index)) for t in labels], np.int32)
    names = [None] * len(index)
    for t, i in index.items():
        names[i] = t
    return ids, names


def map_hits(nlabels, labels, keep):
    """mapHits' result from the distinct relabelled labels of a query's hits (None for NA) and their number: NA when more
    than keep; otherwise the non-NA labels sorted (byte order) and joined with '/', NA when none is left."""
    if nlabels > keep:
        return None
    got = sorted(t for t in labels if t is not None)
    return "/".join(got) if got else None


def match_genera(gen_tax, gen_binom, split_glyph="/"):
    """matchGenera (R/taxonomy.R:175-185); gen_binom is used as a regular expression, as R does."""
    if gen_tax is None or gen_binom is None:
        return False
    if len(gen_tax) == 0 or len(gen_binom) == 0:
        return False
    return (gen_tax == gen_binom or re.search("^" + gen_binom + "[ _" + split_glyph + "]", gen_tax) is not None
            or re.search(split_glyph + gen_binom + "$", gen_tax) is not None)


def merge_species(taxtab, binom):
    """addSpecies' merge (R/taxonomy.R:350-357): -> (array with a Species column appended, names).  The genus column is
    the first named Genus, else the last; rows whose genera do not match get NA in the first column named Species (R's
    character indexing), which is an older column when taxtab already ends in a Species level."""
    tab, names = taxtab
    tab = np.asarray(tab, dtype=object)
    names = list(names)
    if tab.ndim != 2 or tab.shape[0] != len(binom):
        raise api.Dada2bError("dada2b: taxtab must have one row per sequence.")
    gcol = names.index("Genus") if "Genus" in names else tab.shape[1] - 1
    match = [match_genera(tab[i, gcol], binom[i, 0]) for i in range(tab.shape[0])]
    out = np.empty((tab.shape[0], tab.shape[1] + 1), dtype=object)
    out[:, :-1] = tab
    out[:, -1] = binom[:, 1]
    names = names + ["Species"]
    scol = names.index("Species")
    for i, m in enumerate(match):
        if not m:
            out[i, scol] = None
    return out, names


def _merge(taxtab, binom, verbose):
    out, names = merge_species(taxtab, binom)
    if verbose:
        print("Of which", sum(x is not None for x in out[:, names.index("Species")]), "had genera consistent with the input table.", end="")
    return out, names


def _check_queries(seqs):
    if any(len(s) == 0 for s in seqs):
        raise api.Dada2bError("dada2b: empty query sequence; assignSpecies needs non-empty queries.")
    if any(re.search("[^ACGT]", s) for s in seqs):
        raise api.Dada2bError("Non-ACGT characters present in the query sequences.")


class SpeciesDB:
    """A species fasta parsed once with its references resident on the device; assign() / add() as often as needed.
    refFasta: a path, or (ids, seqs) of an already read fasta."""

    def __init__(self, refFasta, device=0):
        ids, refs = read_fasta(refFasta) if isinstance(refFasta, (str, os.PathLike)) else refFasta
        genus, species = parse_species(list(ids))
        self._db = None
        self.device = int(device)
        self.genus_ids, self.genus_names = label_ids(genus)
        self.species_ids, self.species_names = label_ids(species)
        self.nref = len(refs)
        L = _lib()
        r = _Seqs(refs)
        db = C.c_void_p()
        eb = C.create_string_buffer(ERRLEN)
        if L.dada2b_species_db_build(C.byref(r.c), self.genus_ids.ctypes.data, self.species_ids.ctypes.data, self.device, C.byref(db), eb):
            raise api.Dada2bError(eb.value.decode())
        self._db = db
        info = SpeciesDBInfo()
        L.dada2b_species_db_info_get(db, C.byref(info))
        self.info = {k: getattr(info, k) for k, _ in SpeciesDBInfo._fields_ if k != "reserved"}

    def close(self):
        if self._db:
            _lib().dada2b_species_db_free(self._db)
            self._db = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _handle(self):
        if not self._db:
            raise api.Dada2bError("dada2b: the database was closed.")
        return self._db

    def raw(self, seqs, tryRC=False, keep_genus=1, keep_species=1):
        """The native call on a list of strings: dict(nhits, genus_n, genus (id lists, None where cut), species_n, species,
        stats).  keep <= 0: no limit."""
        q = _Seqs(seqs)
        return _native(_lib().dada2b_species_assign, self._handle(), C.byref(q.c), int(bool(tryRC)), int(keep_genus), int(keep_species))

    def hits(self, seqs, tryRC=False):
        """Test hook: every query's distinct hit references, sorted 0-based indices (forward and reverse-complement hits
        combined), and the call's stats."""
        seqs = get_sequences(seqs)
        q = _Seqs(seqs)
        r = _native(_lib().dada2b_test_species_hits, self._handle(), C.byref(q.c), int(bool(tryRC)), hits=True)
        return r["hits"], r["stats"]

    def assign(self, seqs, allowMultiple=False, tryRC=False, n=2000, verbose=False):
        """assignSpecies' result for seqs: (object array [nseq, 2] with None for NA, ["Genus", "Species"]).  n bounds the
        queries of one native call (R's batch size); every call scans all references once."""
        seqs = get_sequences(seqs)
        _check_queries(seqs)
        if int(n) < 1:
            raise api.Dada2bError("dada2b: n must be a positive integer.")
        n = int(n)
        keep = keep_of(allowMultiple)
        ks = 0 if keep == float("inf") else max(int(keep), 1)     # keep <= 0 makes every species NA: cap the lists at 1
        out = np.full((len(seqs), 2), None, dtype=object)
        self.last_stats = []
        for b0 in range(0, len(seqs), n):
            r = self.raw(seqs[b0:b0 + n], tryRC, 1, ks)
            self.last_stats.append(r["stats"])
            for i in range(len(r["nhits"])):
                g, s = r["genus"][i], r["species"][i]
                out[b0 + i, 0] = map_hits(r["genus_n"][i], [] if g is None else [self.genus_names[x] for x in g], 1)
                out[b0 + i, 1] = map_hits(r["species_n"][i], [] if s is None else [self.species_names[x] for x in s], keep)
        if verbose:
            print(sum(x is not None for x in out[:, 1]), "out of", len(seqs), "were assigned to the species level.")
        return out, list(LEVELS)

    def add(self, taxtab, seqs, allowMultiple=False, tryRC=False, n=2000, verbose=False):
        """addSpecies' result: taxtab (the (array, level names) pair of assignTaxonomy, one row per seqs) with a Species
        column appended."""
        return _merge(taxtab, self.assign(seqs, allowMultiple, tryRC, n, verbose)[0], verbose)


def assignSpecies(seqs, refFasta, allowMultiple=False, tryRC=False, n=2000, verbose=False, device=0):
    """R/taxonomy.R:240-289 -> (object array [nseq, 2] with None for NA, ["Genus", "Species"]).  The queries are checked
    before the fasta's format, as in R."""
    seqs = get_sequences(seqs)
    ids, refs = read_fasta(refFasta) if isinstance(refFasta, (str, os.PathLike)) else refFasta
    _check_queries(seqs)
    db = SpeciesDB((ids, refs), device=device)
    try:
        return db.assign(seqs, allowMultiple, tryRC, n, verbose)
    finally:
        db.close()


def addSpecies(taxtab, refFasta, seqs, allowMultiple=False, tryRC=False, n=2000, verbose=False, device=0):
    """R/taxonomy.R:347-360.  taxtab: the (array, level names) pair of assignTaxonomy; seqs: its rows' sequences (R takes
    them from the table's rownames)."""
    seqs = get_sequences(seqs)
    return _merge(taxtab, assignSpecies(seqs, refFasta, allowMultiple, tryRC, n, verbose, device)[0], verbose)

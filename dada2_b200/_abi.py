"""ctypes mirror of include/dada2b.h (struct layouts + marshalling helpers).

Host-side glue only: converts the reference's dada_uniques() argument conventions
(/root/reference/R/dada.R:335-352, src/Rmain.cpp:30-47) to the flat C-ABI structs and
the flat outputs back to a dict shaped like the R list of Rmain.cpp:294.
"""
import ctypes as C
import numpy as np

NA_INTEGER = -2147483648
ERRLEN = 256


class In(C.Structure):
    _fields_ = [("nraw", C.c_int32), ("maxlen", C.c_int32), ("seq_concat", C.c_char_p),
                ("seq_off", C.c_void_p), ("abund", C.c_void_p), ("prior", C.c_void_p),
                ("quals", C.c_void_p), ("err", C.c_void_p), ("Q", C.c_int32)]


class Opts(C.Structure):
    _fields_ = [("match", C.c_int32), ("mismatch", C.c_int32), ("gap", C.c_int32),
                ("use_kmers", C.c_int32), ("kdist_cutoff", C.c_double), ("band_size", C.c_int32),
                ("omegaA", C.c_double), ("omegaP", C.c_double), ("omegaC", C.c_double),
                ("detect_singletons", C.c_int32), ("max_clust", C.c_int32), ("min_fold", C.c_double),
                ("min_hamming", C.c_int32), ("min_abund", C.c_int32), ("use_quals", C.c_int32),
                ("final_consensus", C.c_int32), ("vectorized_alignment", C.c_int32),
                ("homo_gap", C.c_int32), ("multithread", C.c_int32), ("verbose", C.c_int32),
                ("SSE", C.c_int32), ("gapless", C.c_int32), ("greedy", C.c_int32)]


class Out(C.Structure):
    _fields_ = [("nclust", C.c_int32), ("nraw", C.c_int32), ("maxlen", C.c_int32), ("Q", C.c_int32),
                ("n_birth_subs", C.c_int32),
                ("cl_seq_concat", C.c_void_p), ("cl_seq_off", C.c_void_p),
                ("cl_abundance", C.c_void_p), ("cl_n0", C.c_void_p), ("cl_n1", C.c_void_p), ("cl_nunq", C.c_void_p),
                ("cl_pval", C.c_void_p), ("cl_birth_from", C.c_void_p), ("cl_birth_pval", C.c_void_p),
                ("cl_birth_fold", C.c_void_p), ("cl_birth_ham", C.c_void_p), ("cl_birth_qave", C.c_void_p),
                ("bs_pos", C.c_void_p), ("bs_ref", C.c_void_p), ("bs_sub", C.c_void_p), ("bs_qual", C.c_void_p),
                ("bs_clust", C.c_void_p),
                ("subqual", C.c_void_p), ("subqual_ncol", C.c_int32), ("clusterquals", C.c_void_p),
                ("map", C.c_void_p), ("pval", C.c_void_p),
                ("n_align", C.c_int64), ("n_shroud", C.c_int64), ("n_nw", C.c_int64), ("n_gapless", C.c_int64),
                ("nw_cells", C.c_int64), ("n_final_nw", C.c_int64), ("n_rounds", C.c_int32), ("n_shuffles", C.c_int32),
                ("gpu_launches", C.c_int64), ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64),
                ("ms_setup", C.c_double), ("ms_loop", C.c_double), ("ms_final", C.c_double), ("ms_total", C.c_double),
                ("ms_device", C.c_double), ("ms_k_classify", C.c_double), ("ms_k_align_nw", C.c_double),
                ("ms_k_align_gl", C.c_double), ("ms_k_align_final", C.c_double),
                ("n_k_classify", C.c_int32), ("n_k_align_nw", C.c_int32), ("n_k_align_gl", C.c_int32),
                ("n_k_align_final", C.c_int32),
                ("ms_k_prescreen", C.c_double), ("ms_k_nw_bound", C.c_double), ("ms_k_nw_exact", C.c_double), ("ms_k_tail", C.c_double),
                ("n_k_prescreen", C.c_int32), ("n_k_nw_bound", C.c_int32), ("n_k_nw_exact", C.c_int32), ("n_k_tail", C.c_int32),
                ("prescreen_rows", C.c_int64),
                ("ms_k_final_row", C.c_double), ("ms_k_final_diag", C.c_double), ("ms_k_final_gapped", C.c_double),
                ("n_k_final_row", C.c_int32), ("n_k_final_diag", C.c_int32), ("n_k_final_gapped", C.c_int32)]

STAT_FIELDS = ["n_align", "n_shroud", "n_nw", "n_gapless", "nw_cells", "n_final_nw", "n_rounds", "n_shuffles",
               "gpu_launches", "h2d_bytes", "d2h_bytes", "ms_setup", "ms_loop", "ms_final", "ms_total", "ms_device",
               "ms_k_classify", "ms_k_align_nw", "ms_k_align_gl", "ms_k_align_final", "n_k_classify", "n_k_align_nw",
               "n_k_align_gl", "n_k_align_final", "ms_k_prescreen", "ms_k_nw_bound", "ms_k_nw_exact", "ms_k_tail", "n_k_prescreen",
               "n_k_nw_bound", "n_k_nw_exact", "n_k_tail", "prescreen_rows", "ms_k_final_row", "ms_k_final_diag",
               "ms_k_final_gapped", "n_k_final_row", "n_k_final_diag", "n_k_final_gapped"]


# R/dada.R:1-26 defaults, in dada_uniques argument order (R/dada.R:340-352)
DEFAULT_OPTS = dict(match=5, mismatch=-4, gap=-8, use_kmers=True, kdist_cutoff=0.42, band_size=16,
                    omegaA=1e-40, omegaP=1e-4, omegaC=1e-40, detect_singletons=False, max_clust=0,
                    min_fold=1.0, min_hamming=1, min_abund=1, use_quals=True, final_consensus=False,
                    vectorized_alignment=True, homo_gap=-8, multithread=True, verbose=False, SSE=2,
                    gapless=True, greedy=True)


def make_opts(**kw):
    d = dict(DEFAULT_OPTS)
    for k in kw:
        if k not in d:
            raise TypeError("unknown dada_uniques option %r" % k)
    d.update(kw)
    o = Opts()
    for k, _t in Opts._fields_:
        v = d[k]
        setattr(o, k, float(v) if _t is C.c_double else int(v))
    return o


class PackedIn:
    """Keeps the numpy buffers alive for the lifetime of the struct."""

    def __init__(self, seqs, abundances, priors, err, quals):
        nraw = len(seqs)
        if isinstance(seqs, (bytes, bytearray)):
            raise TypeError("seqs must be a sequence of str")
        lens = np.fromiter((len(s) for s in seqs), dtype=np.int64, count=nraw)
        self.off = np.zeros(nraw + 1, dtype=np.int64)
        np.cumsum(lens, out=self.off[1:])
        self.concat = "".join(seqs).encode("ascii")
        self.abund = np.ascontiguousarray(abundances, dtype=np.int32)
        if len(self.abund) != nraw:
            raise ValueError("Sequence and abundance vectors had different lengths.")
        self.prior = None
        if priors is not None:
            self.prior = np.ascontiguousarray(priors, dtype=np.uint8)
            if len(self.prior) != nraw:
                raise ValueError("Sequence and priors vectors had different lengths.")
        self.err = None
        Q = 0
        if err is not None:
            e = np.asarray(err, dtype=np.float64)
            Q = e.shape[1] if e.ndim == 2 else 0
            self.err_rows = e.shape[0] if e.ndim == 2 else 0
            self.err = np.asfortranarray(e)  # column-major 16 x Q
        self.quals = None
        maxlen = 0
        if quals is not None:
            # [nraw, maxlen] row-major == R's maxlen x nraw column-major (position fastest)
            self.quals = np.ascontiguousarray(quals, dtype=np.float64)
            if self.quals.ndim != 2 or self.quals.shape[0] != nraw:       # the C-ABI carries no row count: the library reads nraw rows
                raise ValueError("Qualities must be a matrix with one row per sequence.")
            maxlen = self.quals.shape[1]
        s = In()
        s.nraw = nraw
        s.maxlen = maxlen
        s.seq_concat = self.concat
        s.seq_off = self.off.ctypes.data
        s.abund = self.abund.ctypes.data
        s.prior = self.prior.ctypes.data if self.prior is not None else None
        s.quals = self.quals.ctypes.data if self.quals is not None else None
        s.err = self.err.ctypes.data if self.err is not None else None
        s.Q = Q
        self.struct = s


def _arr(ptr, n, dtype):
    if n <= 0 or not ptr:
        return np.zeros(0, dtype=dtype)
    buf = (C.c_char * (n * np.dtype(dtype).itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype).copy()


def unpack_out(o):
    """Out struct -> dict mirroring list(clustering=, birth_subs=, subqual=, clusterquals=, map=, pval=)."""
    nc, nr = o.nclust, o.nraw
    off = _arr(o.cl_seq_off, nc + 1, np.int64)
    concat = C.string_at(o.cl_seq_concat, int(off[-1])).decode("ascii") if nc else ""
    cl = {"sequence": [concat[off[i]:off[i + 1]] for i in range(nc)]}
    for k in ("abundance", "n0", "n1", "nunq", "birth_from", "birth_ham"):
        cl[k] = _arr(getattr(o, "cl_" + k), nc, np.int32)
    for k in ("pval", "birth_pval", "birth_fold", "birth_qave"):
        cl[k] = _arr(getattr(o, "cl_" + k), nc, np.float64)
    nb = o.n_birth_subs
    bs = {"pos": _arr(o.bs_pos, nb, np.int32), "clust": _arr(o.bs_clust, nb, np.int32),
          "qual": _arr(o.bs_qual, nb, np.float64),
          "ref": [chr(c) for c in _arr(o.bs_ref, nb, np.uint8)],
          "sub": [chr(c) for c in _arr(o.bs_sub, nb, np.uint8)]}
    tc = o.subqual_ncol
    res = {"clustering": cl, "birth_subs": bs,
           "subqual": _arr(o.subqual, 16 * tc, np.int32).reshape((tc, 16)).T.copy(),
           "clusterquals": _arr(o.clusterquals, o.maxlen * nc, np.float64).reshape((nc, o.maxlen)).T.copy(),
           "map": _arr(o.map, nr, np.int32), "pval": _arr(o.pval, nr, np.float64),
           "stats": {k: getattr(o, k) for k in STAT_FIELDS}}
    return res
